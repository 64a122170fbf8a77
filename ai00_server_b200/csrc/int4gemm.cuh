// Projection GEMM over Int4 weight-only quantised matrices, and the quantiser that builds them at load.
//
// Format (B200RWKV_QUANT_INT4; the project's own, beyond the reference's `Quant` enum): Int8's scheme at 4 bits.  Each run of
// 128 consecutive inputs of one output row (a k block) keeps mn = min, rng = max - min (f32), scale = f16(rng / 15),
// min = f16(mn) and every element as q = floor(15 clamp((w - mn) / rng, 0, 1) + 0.5), 0..15 (q = 0 where rng == 0).  The
// GPTQ / AWQ-style asymmetric int4 layout with groups of 128.  tests/int4_oracle.py restates it.
//
// Engine contract: the weight is fma_f16(q, scale, min) with ONE rounding (HFMA2, as Int8's expansion); the tensor cores
// multiply it with the f16 token operand and accumulate in f32.
//
// fp8gemm.cuh's structure: no expansion stage.  The consumer warpgroup LDS's its codes in wgmma's A-fragment order, turns
// them into f16 in its own registers and feeds them to wgmma as the REGISTER A operand (WgmmaRs), with the token operand as
// the shared-memory B descriptor of gemm.cuh.  A code becomes an f16 as Int8's does, without a table: LOP3 puts two nibbles
// into the low bits of two halves with exponent 0x64 ({1024 + q0, 1024 + q1}), HSUB2 1024 (exact), HFMA2 (q, scale, min).
// Every nibble is shifted down to bits 0..3 of its half first, so no scale / 16 product (which would leave the f16 normal
// range for scales below 2^-10) is ever formed.  Producer lane, mbarrier ring, L2 policies, PDL (weights requested before
// griddepcontrol.wait), stream-K SegWalk, gemm_acc_to_rows and gemm_epilogue_tile are gemm.cuh's; a stage block is 8 704 B
// of HBM traffic (one bulk copy) plus the token operand.
//
// Block (128 rows x 128 k): 8 KB of codes [k32 pair 4][consumer thread 128][16 B] | 512 B of (scale, min) f16 pairs.
// Thread t = 32 w + 4 g + c holds, as for FP8, rows 64 h + 16 w + g (+ 8) and k 2c, 2c + 1 (+ 8) of every k16 step; its 16 B
// of one k32 pair are four u32 words, word 2 s + h = k16 step s of the pair, weight half h.  A word holds the half's fragment
// registers a0..a7 as four f16 pairs: pair j (= {a2j, a2j+1}) sits in nibbles p, p + 4 with p = (j >> 1) + 2 (j & 1), so
// (word >> 4p) & 0x000f000f is the pair, and a byte holds elements k and k + 8 of ONE row (low, high nibble): the quantiser's
// warps, one per row, write whole bytes.  A warp's 16-byte LDS are 512 contiguous bytes (no bank conflict), one per two k16
// steps.  The (scale, min) pairs are in the same order: [w 4][g 8][h 2][+8 2]{scale, min}, one 16-byte LDS per thread and
// block.
#pragma once
#include "fp8gemm.cuh"

namespace b200 {

constexpr int INT4_WBYTES = GEMM_BN * GEMM_BK / 2;                   // 8 KB of codes per stage block
constexpr int INT4_BLOCK_BYTES = INT4_WBYTES + Q_PARAM_BYTES;        // 8 704: codes + (scale, min) of its 128 rows
static_assert(INT4_BLOCK_BYTES == Q_NF4_BYTES, "q_block_bytes(QT_INT4)");

// TAILS (int4gemm_tail_kernel, W' plans): a ring slot holds a whole f16 tail block before the token operand
template <int MT, bool TAILS = false>
struct Int4GemmCfg {
    static constexpr int SLOT_W = TAILS ? GEMM_WBYTES : INT4_BLOCK_BYTES;
    static constexpr int STAGE_BYTES = SLOT_W + MT * GEMM_ABYTES;
    static constexpr int NFIT = GEMM_SMEM_BUDGET / STAGE_BYTES;
    static constexpr int NSTAGE = NFIT > 12 ? 12 : NFIT;
    static constexpr int BAR_BYTES = 2 * NSTAGE * 8 + 16;
    static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + BAR_BYTES + 64;
    // k16 steps per MMA group (even: one LDS covers two): two register buffers of KG x 8 registers next to 16 MT accumulators
    static constexpr int KG = MT == 8 ? 2 : 4;
    static_assert(NSTAGE >= 2, "ring needs two stages");
    static_assert(STAGE_BYTES % 128 == 0, "stage blocks stay 128-byte aligned");
    static_assert(KG % 2 == 0 && (GEMM_BK / 16) % KG == 0, "whole k32 pairs per group");
};

// nibble of element (row r, k) of a 128 x 128 tile inside its block (byte = nibble >> 1, high nibble when odd)
__host__ __device__ constexpr int int4_nibble(const int r, const int k) {
    return (((k >> 5) * GEMM_EPI_THREADS + 32 * ((r & 63) >> 4) + 4 * (r & 7) + ((k & 7) >> 1)) * 4 + 2 * ((k >> 4) & 1) + (r >> 6)) * 8 +
           ((k >> 3) & 1) + 2 * ((r >> 3) & 1) + 4 * (k & 1);
}
// byte of row r's (scale, min) pair behind the codes
__host__ __device__ constexpr int int4_param_offset(const int r) {
    return INT4_WBYTES + ((8 * ((r & 63) >> 4) + (r & 7)) * 4 + 2 * (r >> 6) + ((r >> 3) & 1)) * 4;
}

__device__ __forceinline__ uint32_t lop3_and_or(const uint32_t a, const uint32_t b, const uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(b), "r"(c));      // (a & b) | c
    return r;
}

// the two codes in nibbles (sh / 4, sh / 4 + 4) of w -> f16 pair  q * scale + min
__device__ __forceinline__ uint32_t int4_pair(const uint32_t w, const int sh, const __half2 s2, const __half2 m2) {
    const __half2 biased = u32_as_h2(lop3_and_or(w >> sh, 0x000f000fu, 0x64006400u));     // {1024 + q0, 1024 + q1}
    const __half2 q = __hsub2(biased, u32_as_h2(0x64006400u));                             // exact
    return h2_as_u32(__hfma2(q, s2, m2));
}

// one word (8 codes of one k16 step and weight half) -> fragment registers {a0 a1} {a2 a3} {a4 a5} {a6 a7}; row g: s0 / m0,
// row g + 8: s1 / m1
__device__ __forceinline__ void int4x8_to_f16(const uint32_t w, const __half2 s0, const __half2 m0, const __half2 s1, const __half2 m1,
                                              uint32_t (&a)[4]) {
    a[0] = int4_pair(w, 0, s0, m0);
    a[1] = int4_pair(w, 8, s1, m1);
    a[2] = int4_pair(w, 4, s0, m0);
    a[3] = int4_pair(w, 12, s1, m1);
}

// ---------------------------------------------------------------------------------------
// kernel: warps 0-3 consumer warpgroup (conversion + MMA + gemm.cuh epilogue), warp 4 TMA producer
// ---------------------------------------------------------------------------------------
template <int MT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) int4gemm_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = Int4GemmCfg<MT>;
    constexpr int NSTAGE = Cfg::NSTAGE, STAGE_BYTES = Cfg::STAGE_BYTES, KG = Cfg::KG;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int s_last;
    __shared__ __align__(16) float s_x[GEMM_XPOSE_FLOATS];
    const uint32_t ring_base = smem_u32(smem);
    const uint32_t full_bar = ring_base + NSTAGE * STAGE_BYTES;
    const uint32_t empty_bar = full_bar + NSTAGE * 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long TB = p.total_blocks;
    const int G = gridDim.x, cta = blockIdx.x;
    const int b0 = (int)((long long)cta * TB / G);
    const int b1 = (int)((long long)(cta + 1) * TB / G);
    unsigned long long* const tr = (p.trace && cta == 0) ? p.trace : nullptr;

    if (tid == 0) {
        if (tr) tr[0] = globaltimer_ns();
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(full_bar + s * 8, 1);
            mbar_init(empty_bar + s * 8, GEMM_EPI_WARPS);
        }
        mbar_fence_init();
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
                bulk_g2s_hint(ring_base + i * STAGE_BYTES, p.W + (size_t)(b0 + i) * INT4_BLOCK_BYTES, INT4_BLOCK_BYTES, full_bar + i * 8, pol_w);
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
                    bulk_g2s_hint(st, p.W + (size_t)b * INT4_BLOCK_BYTES, INT4_BLOCK_BYTES, fb, pol_w);
                }
                bulk_g2s_hint(st + INT4_BLOCK_BYTES, sg->A + (size_t)kb * A16_KB_HALVES, MT * GEMM_ABYTES, fb, pol_a);
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
    } else {
        // ===================== consumer warpgroup: conversion + MMA + epilogue =====================
        pdl_wait();
        constexpr uint32_t a_lbo = 16 * MT * 16;
        RingPos rp{0, 0u};
        SegWalk w;
        w.init(p, b0, b1);
        while (!w.done()) {
            const int nblk = w.nblk();
            float acc[2][8 * MT];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 8 * MT; ++i) acc[h][i] = 0.f;
            uint32_t a[2][KG][2][4];                   // [register buffer][k16 step of the group][weight half][fragment register]
            int prev_stage = -1;
            for (int i = 0; i < nblk; ++i) {
                mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);
                const uint32_t st = ring_base + rp.stage * STAGE_BYTES;
                const uint32_t ast = st + INT4_BLOCK_BYTES;
                // {scale, min} of rows g, g + 8 (half 0) and 64 + g, 72 + g (half 1) of this thread's fragments
                const uint4 pr = lds128(st + INT4_WBYTES + (uint32_t)(tid >> 2) * 16);
                const uint32_t prw[4] = {pr.x, pr.y, pr.z, pr.w};
                __half2 s2[4], m2[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    s2[j] = u32_as_h2(prmt(prw[j], 0u, 0x1010u));
                    m2[j] = u32_as_h2(prmt(prw[j], 0u, 0x3232u));
                }
#pragma unroll
                for (int g = 0; g < GEMM_BK / 16 / KG; ++g) {
                    uint32_t(&ab)[KG][2][4] = a[g & 1];     // the group that last read this buffer has retired
#pragma unroll
                    for (int s = 0; s < KG; s += 2) {
                        const uint4 c = lds128(st + (uint32_t)((((g * KG + s) >> 1) * GEMM_EPI_THREADS + tid) * 16));
                        int4x8_to_f16(c.x, s2[0], m2[0], s2[1], m2[1], ab[s][0]);
                        int4x8_to_f16(c.y, s2[2], m2[2], s2[3], m2[3], ab[s][1]);
                        int4x8_to_f16(c.z, s2[0], m2[0], s2[1], m2[1], ab[s + 1][0]);
                        int4x8_to_f16(c.w, s2[2], m2[2], s2[3], m2[3], ab[s + 1][1]);
                    }
                    wgmma_fence_operand(acc[0]);
                    wgmma_fence_operand(acc[1]);
                    wgmma_fence();                       // the conversions' register writes before the MMAs that read them
#pragma unroll
                    for (int s = 0; s < KG; ++s) {
                        const uint64_t bdesc = gmma_desc(ast + (g * KG + s) * 2 * a_lbo, a_lbo, GEMM_A_SBO);
#pragma unroll
                        for (int h = 0; h < 2; ++h) WgmmaRs<16 * MT>::mma(acc[h], ab[s][h], bdesc);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                     // the previous group retired: its register buffer may be rewritten
                }
                // every MMA of the previous block has retired: its ring slot goes back
                if (prev_stage >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
                }
                prev_stage = rp.stage;
                rp.advance<NSTAGE>(1);
            }
            wgmma_wait<0>();
            wgmma_fence_operand(acc[0]);
            wgmma_fence_operand(acc[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
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

// W' plans (adapters on quantised layers): code blocks, then f16 tail blocks (GemmParams::tails) with gemm.cuh's shared-memory
// MMAs (fp8gemm.cuh tail_block_mma)
template <int MT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) int4gemm_tail_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = Int4GemmCfg<MT, true>;
    constexpr int NSTAGE = Cfg::NSTAGE, STAGE_BYTES = Cfg::STAGE_BYTES, KG = Cfg::KG;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int s_last;
    __shared__ __align__(16) float s_x[GEMM_XPOSE_FLOATS];
    const uint32_t ring_base = smem_u32(smem);
    const uint32_t full_bar = ring_base + NSTAGE * STAGE_BYTES;
    const uint32_t empty_bar = full_bar + NSTAGE * 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long TB = p.total_blocks;
    const int G = gridDim.x, cta = blockIdx.x;
    const int b0 = (int)((long long)cta * TB / G);
    const int b1 = (int)((long long)(cta + 1) * TB / G);
    unsigned long long* const tr = (p.trace && cta == 0) ? p.trace : nullptr;

    if (tid == 0) {
        if (tr) tr[0] = globaltimer_ns();
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(full_bar + s * 8, 1);
            mbar_init(empty_bar + s * 8, GEMM_EPI_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_launch_dependents();

    if (warp == GEMM_EPI_WARPS) {
        // ===================== producer =====================
        if (lane == 0) tail_producer<MT, NSTAGE, STAGE_BYTES, Cfg::SLOT_W, INT4_BLOCK_BYTES, true>(p, b0, b1, ring_base, full_bar, empty_bar, tr);
    } else {
        // ===================== consumer warpgroup: conversion + MMA + epilogue =====================
        pdl_wait();
        constexpr uint32_t a_lbo = 16 * MT * 16;
        RingPos rp{0, 0u};
        SegWalk w;
        w.init(p, b0, b1);
        while (!w.done()) {
            const int nblk = w.nblk();
            const int nq = max(0, min(nblk, p.kbq[w.seg] - w.kb));     // code blocks first, then f16 tail blocks
            float acc[2][8 * MT];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 8 * MT; ++i) acc[h][i] = 0.f;
            uint32_t a[2][KG][2][4];                   // [register buffer][k16 step of the group][weight half][fragment register]
            int prev_stage = -1;
            for (int i = 0; i < nblk; ++i) {
                mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);
                const uint32_t st = ring_base + rp.stage * STAGE_BYTES;
                const uint32_t ast = st + Cfg::SLOT_W;
                if (i >= nq) {
                    tail_block_mma<MT>(acc, st, ast);
                } else {
                    // {scale, min} of rows g, g + 8 (half 0) and 64 + g, 72 + g (half 1) of this thread's fragments
                    const uint4 pr = lds128(st + INT4_WBYTES + (uint32_t)(tid >> 2) * 16);
                    const uint32_t prw[4] = {pr.x, pr.y, pr.z, pr.w};
                    __half2 s2[4], m2[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        s2[j] = u32_as_h2(prmt(prw[j], 0u, 0x1010u));
                        m2[j] = u32_as_h2(prmt(prw[j], 0u, 0x3232u));
                    }
#pragma unroll
                    for (int g = 0; g < GEMM_BK / 16 / KG; ++g) {
                        uint32_t(&ab)[KG][2][4] = a[g & 1];     // the group that last read this buffer has retired
#pragma unroll
                        for (int s = 0; s < KG; s += 2) {
                            const uint4 c = lds128(st + (uint32_t)((((g * KG + s) >> 1) * GEMM_EPI_THREADS + tid) * 16));
                            int4x8_to_f16(c.x, s2[0], m2[0], s2[1], m2[1], ab[s][0]);
                            int4x8_to_f16(c.y, s2[2], m2[2], s2[3], m2[3], ab[s][1]);
                            int4x8_to_f16(c.z, s2[0], m2[0], s2[1], m2[1], ab[s + 1][0]);
                            int4x8_to_f16(c.w, s2[2], m2[2], s2[3], m2[3], ab[s + 1][1]);
                        }
                        wgmma_fence_operand(acc[0]);
                        wgmma_fence_operand(acc[1]);
                        wgmma_fence();                       // the conversions' register writes before the MMAs that read them
#pragma unroll
                        for (int s = 0; s < KG; ++s) {
                            const uint64_t bdesc = gmma_desc(ast + (g * KG + s) * 2 * a_lbo, a_lbo, GEMM_A_SBO);
#pragma unroll
                            for (int h = 0; h < 2; ++h) WgmmaRs<16 * MT>::mma(acc[h], ab[s][h], bdesc);
                        }
                        wgmma_commit();
                        wgmma_wait<1>();                     // the previous group retired: its register buffer may be rewritten
                    }
                }
                // every MMA of the previous block has retired: its ring slot goes back
                if (prev_stage >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
                }
                prev_stage = rp.stage;
                rp.advance<NSTAGE>(1);
            }
            wgmma_wait<0>();
            wgmma_fence_operand(acc[0]);
            wgmma_fence_operand(acc[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
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
// Quantiser (load time).  One warp per (weight row, 128-wide k block) of rows [n0, n0+N), columns [k0, k0+128 KB) of a
// row-major f16 matrix with row stride ld: lane l holds elements k, k + 8, k + 64, k + 72 with k = 16 (l >> 3) + (l & 7), i.e.
// the two bytes (l and l + 32 of the row's 64 in fragment order) it writes.  quantize_weight_kernel<QT_INT8> with 15 in place
// of 255, spelled with the same _rn intrinsics: the codes must equal tests/int4_oracle.py's bit for bit.
// ---------------------------------------------------------------------------------------
__global__ void quantize_int4_kernel(const __half* __restrict__ src, int ld, int n0, int k0, int N, int tiles, int KB,
                                     uint8_t* __restrict__ dst) {
    const int lane = threadIdx.x & 31;
    const long long nwarp = (long long)tiles * KB * GEMM_BN;
    const int kl = 16 * (lane >> 3) + (lane & 7);
    const int ks[4] = {kl, kl + 8, kl + 64, kl + 72};
    for (long long wi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wi < nwarp; wi += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int r = (int)(wi % GEMM_BN);
        const int kb = (int)((wi / GEMM_BN) % KB);
        const int tile = (int)(wi / ((long long)GEMM_BN * KB));
        const int n = tile * GEMM_BN + r;
        uint8_t* blk = dst + ((size_t)tile * KB + kb) * INT4_BLOCK_BYTES;
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (n < N) {
            const __half* s = src + (size_t)(n0 + n) * ld + k0 + kb * GEMM_BK;
#pragma unroll
            for (int e = 0; e < 4; ++e) x[e] = __half2float(s[ks[e]]);
        }
        float mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3])), mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        const float rng = __fsub_rn(mx, mn);
        uint32_t q[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float t = rng > 0.f ? __fdiv_rn(__fsub_rn(x[e], mn), rng) : 0.f;
            t = fminf(fmaxf(t, 0.f), 1.f);
            q[e] = (uint32_t)floorf(__fadd_rn(__fmul_rn(t, 15.f), 0.5f));
        }
        blk[int4_nibble(r, ks[0]) >> 1] = (uint8_t)(q[0] | q[1] << 4);
        blk[int4_nibble(r, ks[2]) >> 1] = (uint8_t)(q[2] | q[3] << 4);
        if (lane == 0) {
            const __half s = __float2half_rn(__fdiv_rn(rng, 15.f));
            *reinterpret_cast<__half2*>(blk + int4_param_offset(r)) = __halves2half2(s, __float2half_rn(mn));
        }
    }
}

}  // namespace b200
