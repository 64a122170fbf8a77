// Projection GEMM over FP8 (E4M3) weight-only quantised matrices, and the quantiser that builds them at load.
//
// Format (B200RWKV_QUANT_FP8; the project's own, beyond the reference's `Quant` enum): output row n of the FULL [N, K] f16
// matrix keeps one f32 scale s_n = max_k |w_nk| / 448 and every element as the E4M3 code e4m3(w_nk / s_n) (round to nearest
// even, satfinite; 448 is E4M3's largest finite value).  A zero row keeps s_n = 0 and +0 codes.  The scale covers the whole
// row across split-K slices, so a slice's codes are those of the full matrix.  tests/fp8_oracle.py restates it.
//
// Engine contract: every E4M3 value is exactly an f16, so the tensor cores multiply each code's exact value with the f16
// token operand and accumulate in f32; each output is multiplied by s_n in f32 before bias and activation, and before any
// stream-K partial is stored.
//
// Unlike Int8 / NF4 (qgemm.cuh) there is no expansion stage: Hopper converts E4M3 to f16 in hardware (cvt.rn.f16x2.e4m3x2,
// one F2FP per two codes), cheap enough for the consumer warpgroup itself.  So the weights go to wgmma as its REGISTER A
// operand (swap-AB makes A the weight side) and the token operand stays the shared-memory B descriptor of gemm.cuh.  Per
// group of KG k16 steps a thread LDS's its codes, converts them into one of two register buffers and issues the group's
// MMAs; the conversion of the next group overlaps them, and a buffer is rewritten only once the group that read it has
// retired (wgmma.wait_group 1).  A stage block is 16 KB of codes plus the token operand, so the ring holds more stages
// than gemm.cuh's at the same shared memory.  Everything else -- producer lane, mbarrier ring, L2 policies, PDL (weights
// requested before griddepcontrol.wait), stream-K SegWalk, gemm_acc_to_rows, gemm_epilogue_tile -- is gemm.cuh's.
//
// Block (128 rows x 128 k, 16 KB) in wgmma's m64k16 A-fragment order: [k16 step 8][consumer thread 128][weight half 2][8 codes].
// Thread t = 32 w + 4 g + c holds, for half h, rows 64 h + 16 w + g (+ 8) and k 2c, 2c + 1 (+ 8) of the step in register
// order a0..a7, so its 16 codes of one step are ONE 16-byte LDS and a warp's loads are 512 contiguous bytes (no bank
// conflict).  The launch's row scales follow its blocks: [global tile][128 rows] f32 (zero for padding rows).
#pragma once
#include <cuda_fp8.h>

#include "qgemm.cuh"

namespace b200 {

constexpr int FP8_WBYTES = GEMM_BN * GEMM_BK;              // 16 KB of codes per stage block
constexpr int FP8_SCALE_BYTES = GEMM_BN * 4;               // f32 row scales of one tile
constexpr float FP8_E4M3_MAX = 448.f;

// TAILS (fp8gemm_tail_kernel, W' plans): a ring slot holds a whole f16 tail block before the token operand
template <int MT, bool TAILS = false>
struct Fp8GemmCfg {
    static constexpr int SLOT_W = TAILS ? GEMM_WBYTES : FP8_WBYTES;
    static constexpr int STAGE_BYTES = SLOT_W + MT * GEMM_ABYTES;
    static constexpr int NFIT = GEMM_SMEM_BUDGET / STAGE_BYTES;
    static constexpr int NSTAGE = NFIT > 12 ? 12 : NFIT;
    static constexpr int BAR_BYTES = 2 * NSTAGE * 8 + 16;
    static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + BAR_BYTES + 64;
    // k16 steps per MMA group: two register buffers of KG x 8 registers next to the 16 MT accumulator registers
    static constexpr int KG = MT == 8 ? 2 : 4;
    static_assert(NSTAGE >= 2, "ring needs two stages");
    static_assert(STAGE_BYTES % 128 == 0, "stage blocks stay 128-byte aligned");
};

// byte of element (row r, k) of a 128 x 128 tile inside its block
__host__ __device__ constexpr int fp8_code_offset(const int r, const int k) {
    return ((k >> 4) * GEMM_EPI_THREADS + 32 * ((r & 63) >> 4) + 4 * (r & 7) + ((k & 7) >> 1)) * 16 + (r >> 6) * 8 + (k & 1) +
           2 * ((r >> 3) & 1) + 4 * ((k >> 3) & 1);
}

// four E4M3 codes (byte i = element i) -> two f16 pairs {e0, e1}, {e2, e3}
__device__ __forceinline__ void e4m3x4_to_f16(const uint32_t q, uint32_t& lo, uint32_t& hi) {
    asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.rn.f16x2.e4m3x2 %0, l;\n\tcvt.rn.f16x2.e4m3x2 %1, h;\n\t}"
        : "=r"(lo), "=r"(hi)
        : "r"(q));
}

// D[64 x N] += A[64 x 16] * B[N x 16]^T with A in registers (m16k16 fragment per warp: {a0 a1} {a2 a3} {a4 a5} {a6 a7}),
// B K-major through a shared-memory descriptor, f32 accumulator
template <int N>
struct WgmmaRs;
template <>
struct WgmmaRs<16> {
    static __device__ __forceinline__ void mma(float (&d)[8], const uint32_t (&a)[4], uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
    }
};
template <>
struct WgmmaRs<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], const uint32_t (&a)[4], uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
    }
};
template <>
struct WgmmaRs<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
    }
};
template <>
struct WgmmaRs<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
    }
};

// W' plans: the MMAs of one f16 tail block of a ring slot (weights at st, token operand at ast) with the shared-memory A
// descriptors of gemm.cuh, leaving them as the one group in flight (the previous block's MMAs have retired on return)
template <int MT>
__device__ __forceinline__ void tail_block_mma(float (&acc)[2][8 * MT], const uint32_t st, const uint32_t ast) {
    constexpr uint32_t a_lbo = 16 * MT * 16;
    wgmma_fence_operand(acc[0]);
    wgmma_fence_operand(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < GEMM_BK / 16; ++k16) {
        const uint64_t bdesc = gmma_desc(ast + k16 * 2 * a_lbo, a_lbo, GEMM_A_SBO);
#pragma unroll
        for (int h = 0; h < 2; ++h)
            wgmma_f16<16 * MT>(acc[h], gmma_desc(st + h * 8 * GEMM_W_SBO + k16 * 2 * GEMM_W_LBO, GEMM_W_LBO, GEMM_W_SBO), bdesc);
    }
    wgmma_commit();
    wgmma_wait<1>();
}

// ---------------------------------------------------------------------------------------
// kernel: warps 0-3 consumer warpgroup (conversion + MMA + gemm.cuh epilogue), warp 4 TMA producer
// ---------------------------------------------------------------------------------------
template <int MT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) fp8gemm_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = Fp8GemmCfg<MT>;
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
                bulk_g2s_hint(ring_base + i * STAGE_BYTES, p.W + (size_t)(b0 + i) * FP8_WBYTES, FP8_WBYTES, full_bar + i * 8, pol_w);
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
                    bulk_g2s_hint(st, p.W + (size_t)b * FP8_WBYTES, FP8_WBYTES, fb, pol_w);
                }
                bulk_g2s_hint(st + FP8_WBYTES, sg->A + (size_t)kb * A16_KB_HALVES, MT * GEMM_ABYTES, fb, pol_a);
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
        const float* const scales = reinterpret_cast<const float*>(p.W + (size_t)TB * FP8_WBYTES);
        constexpr uint32_t a_lbo = 16 * MT * 16;
        RingPos rp{0, 0u};
        SegWalk w;
        w.init(p, b0, b1);
        while (!w.done()) {
            const int nblk = w.nblk();
            const float scale = scales[(size_t)(p.seg[w.seg].tile_begin + w.tile_local) * GEMM_BN + tid];   // row tid of the tile
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
                const uint32_t ast = st + FP8_WBYTES;
#pragma unroll
                for (int g = 0; g < GEMM_BK / 16 / KG; ++g) {
                    uint32_t(&ab)[KG][2][4] = a[g & 1];     // the group that last read this buffer has retired
#pragma unroll
                    for (int s = 0; s < KG; ++s) {
                        const uint4 c = lds128(st + (uint32_t)(((g * KG + s) * GEMM_EPI_THREADS + tid) * 16));
                        e4m3x4_to_f16(c.x, ab[s][0][0], ab[s][0][1]);
                        e4m3x4_to_f16(c.y, ab[s][0][2], ab[s][0][3]);
                        e4m3x4_to_f16(c.z, ab[s][1][0], ab[s][1][1]);
                        e4m3x4_to_f16(c.w, ab[s][1][2], ab[s][1][3]);
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
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                for (int j = 0; j < 16; ++j) v[mt][j] = __fmul_rn(v[mt][j], scale);
            gemm_epilogue_tile<MT, false>(p, w, cta, G, v, *p.nrows, &s_last, reinterpret_cast<__half*>(s_x));
            w.next();
        }
    }
    __syncthreads();
    if (tid == 0 && tr) tr[7] = globaltimer_ns();
    if (tid == 0 && p.trace) p.trace[8 + 3 * cta + 2] = globaltimer_ns();
}

// W' plans (adapters on quantised layers): code blocks, then f16 tail blocks (GemmParams::tails) with gemm.cuh's shared-memory
// MMAs.  Stream-K partials are summed linearly, so each CTA scales the code part of its accumulator by the row scales before
// its first tail block (or at its end) and adds its tail part unscaled: s_n x W^T + u e^T whichever blocks a CTA holds.
template <int MT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) fp8gemm_tail_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = Fp8GemmCfg<MT, true>;
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
        if (lane == 0) tail_producer<MT, NSTAGE, STAGE_BYTES, Cfg::SLOT_W, FP8_WBYTES, true>(p, b0, b1, ring_base, full_bar, empty_bar, tr);
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
            // the code part of the accumulator times its rows' scales (fragment rows as in gemm_acc_to_rows), before any
            // tail block adds to it and before the partial or the epilogue
            auto scale_codes = [&]() {
                const float* sc = p.scales + (size_t)(p.seg[w.seg].tile_begin + w.tile_local) * GEMM_BN + 16 * warp + (lane >> 2);
                const float s[2][2] = {{sc[0], sc[8]}, {sc[64], sc[72]}};
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 8 * MT; ++i) acc[h][i] = __fmul_rn(acc[h][i], s[h][(i >> 1) & 1]);
            };
            uint32_t a[2][KG][2][4];                   // [register buffer][k16 step of the group][weight half][fragment register]
            int prev_stage = -1;
            for (int i = 0; i < nblk; ++i) {
                mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);
                const uint32_t st = ring_base + rp.stage * STAGE_BYTES;
                const uint32_t ast = st + Cfg::SLOT_W;
                if (i >= nq) {
                    if (i == nq && nq > 0) {
                        wgmma_wait<0>();
                        wgmma_fence_operand(acc[0]);
                        wgmma_fence_operand(acc[1]);
                        scale_codes();
                    }
                    tail_block_mma<MT>(acc, st, ast);
                } else {
#pragma unroll
                    for (int g = 0; g < GEMM_BK / 16 / KG; ++g) {
                        uint32_t(&ab)[KG][2][4] = a[g & 1];     // the group that last read this buffer has retired
#pragma unroll
                        for (int s = 0; s < KG; ++s) {
                            const uint4 c = lds128(st + (uint32_t)(((g * KG + s) * GEMM_EPI_THREADS + tid) * 16));
                            e4m3x4_to_f16(c.x, ab[s][0][0], ab[s][0][1]);
                            e4m3x4_to_f16(c.y, ab[s][0][2], ab[s][0][3]);
                            e4m3x4_to_f16(c.z, ab[s][1][0], ab[s][1][1]);
                            e4m3x4_to_f16(c.w, ab[s][1][2], ab[s][1][3]);
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
            if (nq == nblk) scale_codes();
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
// Quantiser (load time).  One warp per weight row of the launch's `tiles` tiles: the absmax over the whole source row (ld
// columns), then the row's codes for columns [k0, k0 + 128 KB) straight into the fragment-ordered blocks at dst, and its
// scale at scales[row].  f32 arithmetic spelled with _rn intrinsics; the codes must equal tests/fp8_oracle.py's bit for bit.
// ---------------------------------------------------------------------------------------
__global__ void quantize_fp8_kernel(const __half* __restrict__ src, int ld, int n0, int k0, int N, int tiles, int KB,
                                    uint8_t* __restrict__ dst, float* __restrict__ scales) {
    const int lane = threadIdx.x & 31;
    const int nrow = tiles * GEMM_BN;
    for (int n = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5); n < nrow; n += (int)(((long long)gridDim.x * blockDim.x) >> 5)) {
        const int tile = n / GEMM_BN, r = n % GEMM_BN;
        const __half* row = src + (size_t)(n0 + (n < N ? n : 0)) * ld;
        float am = 0.f;
        if (n < N)
            for (int k = lane; k < ld; k += 32) am = fmaxf(am, fabsf(__half2float(row[k])));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
        const float s = __fdiv_rn(am, FP8_E4M3_MAX);
        uint8_t* blk = dst + (size_t)tile * KB * FP8_WBYTES;
        for (int k = lane; k < KB * GEMM_BK; k += 32) {
            uint8_t q = 0;
            if (am > 0.f) q = (uint8_t)__nv_cvt_float_to_fp8(__fdiv_rn(__half2float(row[k0 + k]), s), __NV_SATFINITE, __NV_E4M3);
            blk[(size_t)(k >> 7) * FP8_WBYTES + fp8_code_offset(r, k & 127)] = q;
        }
        if (lane == 0) scales[n] = s;
    }
}

}  // namespace b200
