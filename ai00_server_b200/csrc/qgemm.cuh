// Projection GEMM over weight-only quantised matrices (Int8 / NF4), and the quantisers that build them at load.
//
// Replaces web-rwkv's `quant_mat_int8.wgsl` / `quant_mat_nf4.wgsl` (run once by `ModelBuilder::quant`, reference
// crates/ai00-core/src/lib.rs:465, 484) and its `matmul_{vec,mat}_{int8,nf4}` dispatches inside `Runtime::infer`
// (run.rs:1143) for the first `quant` layers of a model.  Formats (oracle/quant_numpy.py restates them): Int8 = blocks of 128
// consecutive input elements with (min, max) in f16 and round(255 (w - min) / (max - min)) per element; NF4 = blocks of 64
// with absmax in f16 and the index of the nearest NormalFloat4 level per element.
//
// The projection stays the HBM-bound stream of gemm.cuh -- same stream-K split, same consumer warpgroup and epilogue --
// but a stage block is 16.5 KB (Int8) or 8.5 KB (NF4) of HBM traffic instead of 32 KB.  wgmma has no operand format for
// affine u8 or table-coded 4-bit weights, so four expansion warps sit between the TMA ring and the consumer warpgroup:
// thread r owns weight row r of the stage, reads its codes (16-byte LDS), expands them to f16 with two-wide arithmetic and
// writes the row into one of two 32 KB shared-memory buffers in the canonical K-major layout of gemm.cuh; after
// `fence.proxy.async` (generic-proxy stores -> visible to the tensor core's async-proxy reads) an mbarrier arrival hands the
// buffer to the consumer, whose MMAs read it exactly like an f16 weight stage, and the consumer hands it back once those
// MMAs have retired.  Raw blocks are pre-tiled at load so that every shared-memory access of the expansion is a
// conflict-free 16-byte access:
//   Int8 block (128 rows x 128 k): [k16 chunk 8][row 128][16 codes] | [row 128]{f16 scale, f16 min}
//   NF4  block (128 rows x 128 k): [k32 group 4][row 128][16 B = 32 codes, element i of a u32 in bits 4i..4i+3] | [row 128]{f16 absmax k<64, f16 absmax k>=64}
// Int8: codes -> f16 by PRMT into 0x6400|q (= 1024 + q), HSUB2 1024, HFMA2 (q, scale, min): one rounding, bit-identical to the
// oracle's engine contract.  NF4: one LDS of a {level[lo nibble], level[hi nibble]} f16 pair per code byte from a 256-entry table
// replicated per lane (entry-major, 32 KB: every lane stays in its own bank), HMUL2 by absmax.
#pragma once
#include "gemm.cuh"

namespace b200 {

// 3 is the reference's SF4, not implemented (5 is unassigned); FP8: fp8gemm.cuh, Int4: int4gemm.cuh
enum QuantType : int { QT_NONE = 0, QT_INT8 = 1, QT_NF4 = 2, QT_FP8 = 4, QT_INT4 = 6 };

constexpr int Q_PARAM_BYTES = GEMM_BN * 4;                                  // 4 bytes of block parameters per weight row
constexpr int Q_INT8_BYTES = GEMM_BN * GEMM_BK + Q_PARAM_BYTES;             // 16 896
constexpr int Q_NF4_BYTES = GEMM_BN * GEMM_BK / 2 + Q_PARAM_BYTES;          //  8 704
constexpr int Q_DQ_BUFS = 2;                                                // expanded f16 weight buffers in shared memory (32 KB each)
constexpr int Q_DQ_WARPS = 4;
constexpr int Q_DQ_THREADS = Q_DQ_WARPS * 32;                               // = GEMM_BN: one thread per weight row
constexpr int QGEMM_THREADS = GEMM_THREADS + Q_DQ_THREADS;                  // consumer warpgroup + producer + 4 expansion warps
constexpr int Q_LUT_BYTES = 256 * 32 * 4;                                   // NF4: [code byte 256][lane 32] half2

__host__ __device__ constexpr int q_block_bytes(int qt) {
    return qt == QT_INT8 ? Q_INT8_BYTES
         : qt == QT_NF4 || qt == QT_INT4 ? Q_NF4_BYTES            // Int4: 8 KB of codes + (scale, min) per row, as NF4's size
         : qt == QT_FP8 ? GEMM_BN * GEMM_BK : GEMM_WBYTES;
}

__constant__ float c_nf4_levels[16] = {
    -1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f, -0.18477343022823334f,
    -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f,
    0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

template <int MT, int QT>
struct QGemmCfg {
    static constexpr int RAW_W = QT == QT_INT8 ? Q_INT8_BYTES : Q_NF4_BYTES;
    static constexpr int STAGE_BYTES = RAW_W + MT * GEMM_ABYTES;
    static constexpr int LUT = QT == QT_NF4 ? Q_LUT_BYTES : 0;
    static constexpr int NBUF = Q_DQ_BUFS;
    static constexpr int DQ_BYTES = Q_DQ_BUFS * GEMM_WBYTES;
    static constexpr int FIXED = DQ_BYTES + LUT;
    static constexpr int NFIT = (GEMM_SMEM_BUDGET - FIXED) / STAGE_BYTES;
    static constexpr int NSTAGE = NFIT > 12 ? 12 : NFIT;
    static constexpr int BAR_BYTES = (2 * NSTAGE + 2 * NBUF) * 8 + 16;
    static constexpr int SMEM_BYTES = FIXED + NSTAGE * STAGE_BYTES + BAR_BYTES + 64;
    static_assert(NSTAGE >= 2, "ring needs two stages");
    static_assert(RAW_W % 128 == 0 && STAGE_BYTES % 128 == 0, "stage blocks stay 128-byte aligned");
};

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}
__device__ __forceinline__ uint32_t h2_as_u32(const __half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ __half2 u32_as_h2(const uint32_t u) { return *reinterpret_cast<const __half2*>(&u); }

// two Int8 codes (bytes `sel` of w) -> f16 pair  q * scale + min
__device__ __forceinline__ uint32_t int8_pair(const uint32_t w, const uint32_t sel, const __half2 s2, const __half2 m2) {
    const __half2 biased = u32_as_h2(prmt(w, 0x64646464u, sel));               // {1024 + q0, 1024 + q1}
    const __half2 q = __hsub2(biased, u32_as_h2(0x64006400u));                 // exact
    return h2_as_u32(__hfma2(q, s2, m2));
}

// ---------------------------------------------------------------------------------------
// Quantised W' plans (adapters on quantised layers): the launch's linear stage blocks walked one at a time, and the producer
// lane of the tail kernels.  A tile's f16 tail blocks follow its code blocks in the block sequence, so the stream-K cuts,
// SegWalk and the epilogue are unchanged; only where a block's weights live differs (GemmParams::tails).
// ---------------------------------------------------------------------------------------
struct TailPos {
    int seg, tile, kb;
    __device__ __forceinline__ void init(const GemmParams& p, const int b) {
        seg = gemm_find_seg(p, b);
        const GemmSeg& sg = p.seg[seg];
        tile = (b - sg.blk_begin) / sg.KB;
        kb = b - sg.blk_begin - tile * sg.KB;
    }
    __device__ __forceinline__ void next(const GemmParams& p) {
        if (++kb < p.seg[seg].KB) return;
        kb = 0;
        if (++tile < p.seg[seg].tiles) return;
        tile = 0;
        if (seg + 1 < p.nseg) ++seg;
    }
    __device__ __forceinline__ bool tail(const GemmParams& p) const { return kb >= p.kbq[seg]; }
    __device__ __forceinline__ const uint8_t* tail_src(const GemmParams& p) const {
        const int q = p.kbq[seg];
        return p.tails + ((size_t)p.tblk[seg] + (size_t)tile * (p.seg[seg].KB - q) + (kb - q)) * GEMM_WBYTES;
    }
    // code block of QB bytes
    __device__ __forceinline__ const uint8_t* code_src(const GemmParams& p, const int QB) const {
        return p.W + ((size_t)p.qblk[seg] + (size_t)tile * p.kbq[seg] + kb) * QB;
    }
};

// The producer lane of gemm.cuh for W' plans: code blocks of QB bytes and, with TAIL_IN_RING, the 32 KB tail blocks go to the
// ring slot (SLOT_W bytes), the token operand after them; without it a tail block's slot receives the token operand only.
template <int MT, int NSTAGE, int STAGE_BYTES, int SLOT_W, int QB, bool TAIL_IN_RING>
__device__ __forceinline__ void tail_producer(const GemmParams& p, const int b0, const int b1, const uint32_t ring_base,
                                              const uint32_t full_bar, const uint32_t empty_bar, unsigned long long* tr) {
    static_assert(!TAIL_IN_RING || SLOT_W >= GEMM_WBYTES, "a tail block fits its ring slot");
    const uint64_t pol_w = l2_policy_evict_first();
    const uint64_t pol_a = l2_policy_evict_last();
    auto weights = [&](const TailPos& q, const uint32_t st, const uint32_t fb) {
        const bool tail = q.tail(p);
        const int wb = tail ? (TAIL_IN_RING ? GEMM_WBYTES : 0) : QB;
        mbar_expect_tx(fb, wb + MT * GEMM_ABYTES);
        if (wb) bulk_g2s_hint(st, tail ? q.tail_src(p) : q.code_src(p, QB), wb, fb, pol_w);
    };
    TailPos pos;
    pos.init(p, b0);
    TailPos pre = pos;
    const int npre = min(b1 - b0, NSTAGE);
    for (int i = 0; i < npre; ++i, pre.next(p)) weights(pre, ring_base + i * STAGE_BYTES, full_bar + i * 8);    // before the wait, as gemm.cuh
    pdl_wait();
    if (tr) tr[2] = globaltimer_ns();
    int stage = 0;
    uint32_t ephase = 1;
    for (int b = b0, it = 0; b < b1; ++b, ++it, pos.next(p)) {
        const uint32_t st = ring_base + stage * STAGE_BYTES;
        const uint32_t fb = full_bar + stage * 8;
        if (it >= NSTAGE) {
            mbar_wait(empty_bar + stage * 8, ephase, 14);
            weights(pos, st, fb);
        }
        bulk_g2s_hint(st + SLOT_W, p.seg[pos.seg].A + (size_t)pos.kb * A16_KB_HALVES, MT * GEMM_ABYTES, fb, pol_a);
        if (++stage == NSTAGE) { stage = 0; ephase ^= 1; }
    }
}

// ---------------------------------------------------------------------------------------
// expansion role: 128 threads, thread r = weight row r of every stage block, into the canonical layout of gemm.cuh
// ---------------------------------------------------------------------------------------
template <int QT>
__device__ __forceinline__ void q_expand_block(const uint32_t raw, const uint32_t dq, const uint32_t lut, const int r, const int lane) {
    if (QT == QT_INT8) {
        const uint32_t sm = lds32(raw + GEMM_BN * GEMM_BK + r * 4);            // lo = scale, hi = min
        const __half2 s2 = u32_as_h2(prmt(sm, 0u, 0x1010u));
        const __half2 m2 = u32_as_h2(prmt(sm, 0u, 0x3232u));
        uint4 q[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) q[c] = lds128(raw + (uint32_t)(c * GEMM_BN + r) * 16);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            uint4 o0, o1;      // k = 16c .. 16c+7 and 16c+8 .. 16c+15
            o0.x = int8_pair(q[c].x, 0x4140u, s2, m2); o0.y = int8_pair(q[c].x, 0x4342u, s2, m2);
            o0.z = int8_pair(q[c].y, 0x4140u, s2, m2); o0.w = int8_pair(q[c].y, 0x4342u, s2, m2);
            o1.x = int8_pair(q[c].z, 0x4140u, s2, m2); o1.y = int8_pair(q[c].z, 0x4342u, s2, m2);
            o1.z = int8_pair(q[c].w, 0x4140u, s2, m2); o1.w = int8_pair(q[c].w, 0x4342u, s2, m2);
            sts128(dq + (uint32_t)((2 * c) * GEMM_BN + r) * 16, o0);
            sts128(dq + (uint32_t)((2 * c + 1) * GEMM_BN + r) * 16, o1);
        }
    } else {
        const uint32_t am = lds32(raw + GEMM_BN * GEMM_BK / 2 + r * 4);        // lo = absmax of k < 64, hi = of k >= 64
        const uint32_t lut_lane = lut + lane * 4;
#pragma unroll
        for (int g = 0; g < 4; ++g) {                                          // k = 32g .. 32g+31
            const __half2 a2 = u32_as_h2(prmt(am, 0u, g < 2 ? 0x1010u : 0x3232u));
            const uint4 v = lds128(raw + (uint32_t)(g * GEMM_BN + r) * 16);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {                                      // k8 chunk 4g + j
                uint4 o;
                o.x = h2_as_u32(__hmul2(u32_as_h2(lds32(lut_lane + ((w[j] & 0xffu) << 7))), a2));
                o.y = h2_as_u32(__hmul2(u32_as_h2(lds32(lut_lane + (((w[j] >> 8) & 0xffu) << 7))), a2));
                o.z = h2_as_u32(__hmul2(u32_as_h2(lds32(lut_lane + (((w[j] >> 16) & 0xffu) << 7))), a2));
                o.w = h2_as_u32(__hmul2(u32_as_h2(lds32(lut_lane + ((w[j] >> 24) << 7))), a2));
                sts128(dq + (uint32_t)((4 * g + j) * GEMM_BN + r) * 16, o);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// kernel: warps 0-3 consumer warpgroup (MMA + gemm.cuh epilogue), warp 4 TMA producer, warps 5-8 expansion
// ---------------------------------------------------------------------------------------
template <int MT, int QT>
__global__ void __launch_bounds__(QGEMM_THREADS, 1) qgemm_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = QGemmCfg<MT, QT>;
    constexpr int NBUF = Cfg::NBUF;
    constexpr int NSTAGE = Cfg::NSTAGE, STAGE_BYTES = Cfg::STAGE_BYTES, RAW_W = Cfg::RAW_W;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int s_last;
    __shared__ __align__(16) float s_x[GEMM_XPOSE_FLOATS];
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t dq_base = smem_base;
    const uint32_t lut_base = dq_base + Cfg::DQ_BYTES;
    const uint32_t ring_base = lut_base + Cfg::LUT;
    const uint32_t full_bar = ring_base + NSTAGE * STAGE_BYTES;
    const uint32_t empty_bar = full_bar + NSTAGE * 8;
    const uint32_t dfull_bar = empty_bar + NSTAGE * 8;
    const uint32_t dfree_bar = dfull_bar + NBUF * 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long TB = p.total_blocks;
    const int G = gridDim.x, cta = blockIdx.x;
    const int b0 = (int)((long long)cta * TB / G);
    const int b1 = (int)((long long)(cta + 1) * TB / G);
    unsigned long long* const tr = (p.trace && cta == 0) ? p.trace : nullptr;
    constexpr int EXP_WARP0 = GEMM_THREADS / 32;

    if (tid == 0) {
        if (tr) tr[0] = globaltimer_ns();
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(full_bar + s * 8, 1);
            mbar_init(empty_bar + s * 8, GEMM_EPI_WARPS);
        }
        for (int s = 0; s < NBUF; ++s) {
            mbar_init(dfull_bar + s * 8, Q_DQ_WARPS);          // one arrival per expansion warp
            mbar_init(dfree_bar + s * 8, GEMM_EPI_WARPS);
        }
        mbar_fence_init();
    }
    if (QT == QT_NF4 && warp >= EXP_WARP0) {
        // level-pair table, one copy per lane: entry (byte, lane) = {level[byte & 15], level[byte >> 4]}
        const int t = tid - GEMM_THREADS;
        for (int i = t; i < 256 * 32; i += Q_DQ_THREADS) {
            const int byte = i >> 5;
            const __half2 e = __halves2half2(__float2half_rn(c_nf4_levels[byte & 15]), __float2half_rn(c_nf4_levels[byte >> 4]));
            *reinterpret_cast<__half2*>(smem + (lut_base - smem_base) + (size_t)i * 4) = e;
        }
    }
    __syncthreads();
    pdl_launch_dependents();

    if (warp == GEMM_EPI_WARPS) {
        // ===================== producer =====================
        if (lane == 0) {
            const uint64_t pol_w = l2_policy_evict_first();
            const uint64_t pol_a = l2_policy_evict_last();
            const int npre = min(b1 - b0, NSTAGE);
            for (int i = 0; i < npre; ++i) {          // weights never change: requested before the preceding kernel has finished
                mbar_expect_tx(full_bar + i * 8, STAGE_BYTES);
                bulk_g2s_hint(ring_base + i * STAGE_BYTES, p.W + (size_t)(b0 + i) * RAW_W, RAW_W, full_bar + i * 8, pol_w);
            }
            pdl_wait();
            if (tr) tr[2] = globaltimer_ns();
            int seg = gemm_find_seg(p, b0);
            const GemmSeg* sg = &p.seg[seg];
            int kb = (b0 - sg->blk_begin) % sg->KB;
            int blocks_left_in_seg = sg->blk_begin + sg->tiles * sg->KB - b0;
            int stage = 0;
            uint32_t ephase = 1;
            for (int b = b0, it = 0; b < b1; ++b, ++it) {
                const uint32_t st = ring_base + stage * STAGE_BYTES;
                const uint32_t fb = full_bar + stage * 8;
                if (it >= NSTAGE) {
                    mbar_wait(empty_bar + stage * 8, ephase, 14);
                    mbar_expect_tx(fb, STAGE_BYTES);
                    bulk_g2s_hint(st, p.W + (size_t)b * RAW_W, RAW_W, fb, pol_w);
                }
                bulk_g2s_hint(st + RAW_W, sg->A + (size_t)kb * A16_KB_HALVES, MT * GEMM_ABYTES, fb, pol_a);
                if (++stage == NSTAGE) { stage = 0; ephase ^= 1; }
                if (++kb == sg->KB) kb = 0;
                if (--blocks_left_in_seg == 0 && b + 1 < b1) {
                    ++seg;
                    sg = &p.seg[seg];
                    kb = 0;
                    blocks_left_in_seg = sg->tiles * sg->KB;
                }
            }
        }
    } else if (warp >= EXP_WARP0) {
        // ===================== expansion: 4 warps =====================
        const int r = tid - GEMM_THREADS;
        RingPos rp{0, 0u};
        for (int b = b0, it = 0; b < b1; ++b, ++it) {
            const int d = it % NBUF;
            const int u = it / NBUF;
            mbar_wait(full_bar + rp.stage * 8, rp.phase, 16);
            if (u > 0) mbar_wait(dfree_bar + d * 8, (unsigned)(u - 1) & 1u, 17);          // the MMAs that read this buffer retired
            q_expand_block<QT>(ring_base + rp.stage * STAGE_BYTES, dq_base + d * GEMM_WBYTES, lut_base, r, lane);
            fence_proxy_async();                     // generic-proxy stores -> visible to the tensor core's async-proxy reads
            __syncwarp();                            // the other lanes' (fenced) stores happen before lane 0's release
            if (lane == 0) mbar_arrive(dfull_bar + d * 8);
            rp.advance<NSTAGE>(1);
        }
    } else {
        // ===================== consumer warpgroup: MMA + epilogue =====================
        pdl_wait();
        constexpr uint32_t a_lbo = 16 * MT * 16;
        RingPos rp{0, 0u};
        int it = 0;
        SegWalk w;
        w.init(p, b0, b1);
        while (!w.done()) {
            const int nblk = w.nblk();
            float acc[2][8 * MT];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 8 * MT; ++i) acc[h][i] = 0.f;
            int prev_stage = -1, prev_d = -1;
            for (int i = 0; i < nblk; ++i, ++it) {
                const int d = it % NBUF;
                mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);                     // token operand landed
                mbar_wait(dfull_bar + d * 8, (unsigned)(it / NBUF) & 1u, 15);         // weights expanded
                const uint32_t wst = dq_base + d * GEMM_WBYTES;
                const uint32_t ast = ring_base + rp.stage * STAGE_BYTES + RAW_W;
                wgmma_fence_operand(acc[0]);
                wgmma_fence_operand(acc[1]);
                wgmma_fence();
#pragma unroll
                for (int k16 = 0; k16 < GEMM_BK / 16; ++k16) {
                    const uint64_t bdesc = gmma_desc(ast + k16 * 2 * a_lbo, a_lbo, GEMM_A_SBO);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        wgmma_f16<16 * MT>(acc[h], gmma_desc(wst + h * 8 * GEMM_W_SBO + k16 * 2 * GEMM_W_LBO, GEMM_W_LBO, GEMM_W_SBO), bdesc);
                }
                wgmma_commit();
                wgmma_wait<1>();                     // the previous block's MMAs retired: its ring slot and buffer go back
                if (prev_stage >= 0) {
                    __syncwarp();
                    if (lane == 0) { mbar_arrive(empty_bar + prev_stage * 8); mbar_arrive(dfree_bar + prev_d * 8); }
                }
                prev_stage = rp.stage;
                prev_d = d;
                rp.advance<NSTAGE>(1);
            }
            wgmma_wait<0>();
            wgmma_fence_operand(acc[0]);
            wgmma_fence_operand(acc[1]);
            __syncwarp();
            if (lane == 0) { mbar_arrive(empty_bar + prev_stage * 8); mbar_arrive(dfree_bar + prev_d * 8); }
            float v[MT][16];
            gemm_acc_to_rows<MT>(acc, v, s_x);
            gemm_epilogue_tile<MT, false>(p, w, cta, G, v, *p.nrows, &s_last, reinterpret_cast<__half*>(s_x));
            w.next();
        }
    }
    __syncthreads();
    if (tid == 0 && tr) tr[7] = globaltimer_ns();
    if (tid == 0 && p.trace) p.trace[8 + 3 * cta + 2] = globaltimer_ns();
}

// W' plans (adapters on quantised layers): qgemm_kernel over code blocks and f16 tail blocks (GemmParams::tails).  A tail
// block's ring slot holds only its token operand; the expansion warps copy the tail block from global memory into the
// hand-off buffer instead of expanding codes, and the consumer reads it as any other.  The ring keeps the base kernel's size.
template <int MT, int QT>
__global__ void __launch_bounds__(QGEMM_THREADS, 1) qgemm_tail_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = QGemmCfg<MT, QT>;
    constexpr int NBUF = Cfg::NBUF;
    constexpr int NSTAGE = Cfg::NSTAGE, STAGE_BYTES = Cfg::STAGE_BYTES, RAW_W = Cfg::RAW_W;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int s_last;
    __shared__ __align__(16) float s_x[GEMM_XPOSE_FLOATS];
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t dq_base = smem_base;
    const uint32_t lut_base = dq_base + Cfg::DQ_BYTES;
    const uint32_t ring_base = lut_base + Cfg::LUT;
    const uint32_t full_bar = ring_base + NSTAGE * STAGE_BYTES;
    const uint32_t empty_bar = full_bar + NSTAGE * 8;
    const uint32_t dfull_bar = empty_bar + NSTAGE * 8;
    const uint32_t dfree_bar = dfull_bar + NBUF * 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long TB = p.total_blocks;
    const int G = gridDim.x, cta = blockIdx.x;
    const int b0 = (int)((long long)cta * TB / G);
    const int b1 = (int)((long long)(cta + 1) * TB / G);
    unsigned long long* const tr = (p.trace && cta == 0) ? p.trace : nullptr;
    constexpr int EXP_WARP0 = GEMM_THREADS / 32;

    if (tid == 0) {
        if (tr) tr[0] = globaltimer_ns();
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(full_bar + s * 8, 1);
            mbar_init(empty_bar + s * 8, GEMM_EPI_WARPS);
        }
        for (int s = 0; s < NBUF; ++s) {
            mbar_init(dfull_bar + s * 8, Q_DQ_WARPS);          // one arrival per expansion warp
            mbar_init(dfree_bar + s * 8, GEMM_EPI_WARPS);
        }
        mbar_fence_init();
    }
    if (QT == QT_NF4 && warp >= EXP_WARP0) {
        // level-pair table, one copy per lane: entry (byte, lane) = {level[byte & 15], level[byte >> 4]}
        const int t = tid - GEMM_THREADS;
        for (int i = t; i < 256 * 32; i += Q_DQ_THREADS) {
            const int byte = i >> 5;
            const __half2 e = __halves2half2(__float2half_rn(c_nf4_levels[byte & 15]), __float2half_rn(c_nf4_levels[byte >> 4]));
            *reinterpret_cast<__half2*>(smem + (lut_base - smem_base) + (size_t)i * 4) = e;
        }
    }
    __syncthreads();
    pdl_launch_dependents();

    if (warp == GEMM_EPI_WARPS) {
        // ===================== producer =====================
        if (lane == 0) tail_producer<MT, NSTAGE, STAGE_BYTES, RAW_W, RAW_W, false>(p, b0, b1, ring_base, full_bar, empty_bar, tr);
    } else if (warp >= EXP_WARP0) {
        // ===================== expansion: 4 warps =====================
        const int r = tid - GEMM_THREADS;
        RingPos rp{0, 0u};
        TailPos pos;
        pos.init(p, b0);
        for (int b = b0, it = 0; b < b1; ++b, ++it) {
            const int d = it % NBUF;
            const int u = it / NBUF;
            mbar_wait(full_bar + rp.stage * 8, rp.phase, 16);
            if (u > 0) mbar_wait(dfree_bar + d * 8, (unsigned)(u - 1) & 1u, 17);          // the MMAs that read this buffer retired
            if (pos.tail(p)) {
                // 2048 16-byte chunks, already in the buffer's layout: 4 loads in flight per thread at a time (more spill at MT = 8)
                const uint4* src = reinterpret_cast<const uint4*>(pos.tail_src(p));
#pragma unroll
                for (int j0 = 0; j0 < GEMM_WBYTES / 16 / Q_DQ_THREADS; j0 += 4) {
                    uint4 v[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[j] = __ldg(src + (j0 + j) * Q_DQ_THREADS + r);
#pragma unroll
                    for (int j = 0; j < 4; ++j) sts128(dq_base + d * GEMM_WBYTES + (uint32_t)((j0 + j) * Q_DQ_THREADS + r) * 16, v[j]);
                }
            } else {
                q_expand_block<QT>(ring_base + rp.stage * STAGE_BYTES, dq_base + d * GEMM_WBYTES, lut_base, r, lane);
            }
            fence_proxy_async();                     // generic-proxy stores -> visible to the tensor core's async-proxy reads
            __syncwarp();                            // the other lanes' (fenced) stores happen before lane 0's release
            if (lane == 0) mbar_arrive(dfull_bar + d * 8);
            rp.advance<NSTAGE>(1);
            pos.next(p);
        }
    } else {
        // ===================== consumer warpgroup: MMA + epilogue =====================
        pdl_wait();
        constexpr uint32_t a_lbo = 16 * MT * 16;
        RingPos rp{0, 0u};
        int it = 0;
        SegWalk w;
        w.init(p, b0, b1);
        while (!w.done()) {
            const int nblk = w.nblk();
            float acc[2][8 * MT];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 8 * MT; ++i) acc[h][i] = 0.f;
            int prev_stage = -1, prev_d = -1;
            for (int i = 0; i < nblk; ++i, ++it) {
                const int d = it % NBUF;
                mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);                     // token operand landed
                mbar_wait(dfull_bar + d * 8, (unsigned)(it / NBUF) & 1u, 15);         // weights expanded
                const uint32_t wst = dq_base + d * GEMM_WBYTES;
                const uint32_t ast = ring_base + rp.stage * STAGE_BYTES + RAW_W;
                wgmma_fence_operand(acc[0]);
                wgmma_fence_operand(acc[1]);
                wgmma_fence();
#pragma unroll
                for (int k16 = 0; k16 < GEMM_BK / 16; ++k16) {
                    const uint64_t bdesc = gmma_desc(ast + k16 * 2 * a_lbo, a_lbo, GEMM_A_SBO);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        wgmma_f16<16 * MT>(acc[h], gmma_desc(wst + h * 8 * GEMM_W_SBO + k16 * 2 * GEMM_W_LBO, GEMM_W_LBO, GEMM_W_SBO), bdesc);
                }
                wgmma_commit();
                wgmma_wait<1>();                     // the previous block's MMAs retired: its ring slot and buffer go back
                if (prev_stage >= 0) {
                    __syncwarp();
                    if (lane == 0) { mbar_arrive(empty_bar + prev_stage * 8); mbar_arrive(dfree_bar + prev_d * 8); }
                }
                prev_stage = rp.stage;
                prev_d = d;
                rp.advance<NSTAGE>(1);
            }
            wgmma_wait<0>();
            wgmma_fence_operand(acc[0]);
            wgmma_fence_operand(acc[1]);
            __syncwarp();
            if (lane == 0) { mbar_arrive(empty_bar + prev_stage * 8); mbar_arrive(dfree_bar + prev_d * 8); }
            float v[MT][16];
            gemm_acc_to_rows<MT>(acc, v, s_x);
            gemm_epilogue_tile<MT, false>(p, w, cta, G, v, *p.nrows, &s_last, reinterpret_cast<__half*>(s_x));
            w.next();
        }
    }
    __syncthreads();
    if (tid == 0 && tr) tr[7] = globaltimer_ns();
    if (tid == 0 && p.trace) p.trace[8 + 3 * cta + 2] = globaltimer_ns();
}


// ---------------------------------------------------------------------------------------
// Quantisers (load time).  One warp per (weight row, 128-wide k block): lane l holds elements 4l .. 4l+3.
// Source: rows [n0, n0+N), columns [k0, k0+K) of a row-major f16 matrix with row stride ld; K % 128 == 0.
// f32 arithmetic is spelled with the _rn intrinsics so that no multiply-add is contracted: the codes must equal
// oracle/quant_numpy.py's bit for bit.
// ---------------------------------------------------------------------------------------
template <int QT>
__global__ void quantize_weight_kernel(const __half* __restrict__ src, int ld, int n0, int k0, int N, int tiles, int KB,
                                       uint8_t* __restrict__ dst) {
    constexpr int BLK = QT == QT_INT8 ? Q_INT8_BYTES : Q_NF4_BYTES;
    const int lane = threadIdx.x & 31;
    const long long nwarp = (long long)tiles * KB * GEMM_BN;
    for (long long wi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wi < nwarp; wi += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int r = (int)(wi % GEMM_BN);
        const int kb = (int)((wi / GEMM_BN) % KB);
        const int tile = (int)(wi / ((long long)GEMM_BN * KB));
        const int n = tile * GEMM_BN + r;
        uint8_t* blk = dst + ((size_t)tile * KB + kb) * BLK;
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (n < N) {
            const __half* s = src + (size_t)(n0 + n) * ld + k0 + kb * GEMM_BK + 4 * lane;
#pragma unroll
            for (int e = 0; e < 4; ++e) x[e] = __half2float(s[e]);
        }
        if (QT == QT_INT8) {
            float mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3])), mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3]));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            }
            const float rng = __fsub_rn(mx, mn);
            uint32_t code = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float t = rng > 0.f ? __fdiv_rn(__fsub_rn(x[e], mn), rng) : 0.f;
                t = fminf(fmaxf(t, 0.f), 1.f);
                const uint32_t q = (uint32_t)floorf(__fadd_rn(__fmul_rn(t, 255.f), 0.5f));
                code |= q << (8 * e);
            }
            const int k = 4 * lane;
            *reinterpret_cast<uint32_t*>(blk + (size_t)((k >> 4) * GEMM_BN + r) * 16 + (k & 15)) = code;
            if (lane == 0) {
                const __half s = __float2half_rn(__fdiv_rn(rng, 255.f));
                *reinterpret_cast<__half2*>(blk + GEMM_BN * GEMM_BK + r * 4) = __halves2half2(s, __float2half_rn(mn));
            }
        } else {
            float am = fmaxf(fmaxf(fabsf(x[0]), fabsf(x[1])), fmaxf(fabsf(x[2]), fabsf(x[3])));
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));      // 16 lanes = one 64-wide block
            uint32_t code = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                uint32_t best = 7;
                if (am > 0.f) {
                    const float t = __fdiv_rn(x[e], am);
                    float bd = 3.0e38f;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const float dd = fabsf(__fsub_rn(t, c_nf4_levels[i]));
                        if (dd < bd) { bd = dd; best = i; }
                    }
                }
                code |= best << (4 * e);
            }
            const int k = 4 * lane;       // 4 codes = 2 bytes at byte (k % 32) / 2 of the row's k32 group
            *reinterpret_cast<uint16_t*>(blk + (size_t)((k >> 5) * GEMM_BN + r) * 16 + ((k & 31) >> 1)) = (uint16_t)code;
            const float am_hi = __shfl_sync(0xffffffffu, am, 16);
            if (lane == 0) *reinterpret_cast<__half2*>(blk + GEMM_BN * GEMM_BK / 2 + r * 4) = __halves2half2(__float2half_rn(am), __float2half_rn(am_hi));
        }
    }
}

}  // namespace b200
