// Skinny projection GEMM for decode:  Y[T, N] = X[T, K] (f16) * W[N, K]^T (f16), f32 accumulate.
//
// Replaces web-rwkv's WGSL `matmul_vec_fp16` / `matmul_mat_fp16` dispatches that the reference
// reaches through `Runtime::infer` (reference crates/ai00-core/src/run.rs:1143): the R/K/V/G/O,
// channel-mix, LoRA and head projections (SURVEY.md §2.2 K3-K5, K8-K10).
//
// HBM-bound by construction (T <= 64 rows per pass, each weight byte is used once per step), so
// the design is about keeping ~200 KB of weight bytes in flight per SM and never stalling the
// stream.  The tensor work is on Hopper's warpgroup MMA (wgmma):
//   * swap-AB: the WEIGHT tile (128 rows = two m64 MMAs) is the M operand, the token tile is the N = 16 MT operand,
//     both read from shared memory through descriptors; the f32 accumulator lives in the registers of the consumer
//     warpgroup, eight k16 steps per 32 KB stage;
//   * weights are re-tiled ONCE at load into 32 KB stage blocks (128 output rows x 128 k) already
//     in the canonical K-major / no-swizzle shared-memory layout, so a pipeline stage is ONE
//     contiguous 1-D bulk TMA copy (cp.async.bulk -> UBLKCP) that the tensor core reads in place;
//     activations use the matching A16 layout (common.cuh): one bulk copy of MT x 4 KB per stage (the
//     issue rate of bulk copies is what sizes the stage);
//   * warp roles: one TMA producer lane drives a 3-6 stage mbarrier ring; the consumer warpgroup (4 warps) issues the
//     MMAs of a stage, keeps one stage of MMAs in flight and releases each slot when its MMAs retire, then runs the
//     epilogue of the tile from its registers while the producer keeps the ring full;
//   * work is split stream-K style: the launch's stage blocks (all segments, all tiles) form one
//     linear sequence cut into equal contiguous ranges, so every SM streams the same number of
//     bytes whatever the matrix shapes;
//   * tiles cut across CTAs are reduced deterministically: each contributor writes its partial
//     tile to an L2-resident workspace, bumps a per-tile counter, and the LAST arriver sums the
//     partials in fixed slot order and runs the fused epilogue (no spinning, no float atomics);
//   * a launch carries up to 8 "segments" (independent matrices, own input, K and epilogue) so
//     R/K/V/G + decay-LoRA, or the five ddlerp LoRAs, go out as ONE kernel.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace b200 {

constexpr int GEMM_BN = 128;                 // output rows (weight rows) per tile = two wgmma M = 64
constexpr int GEMM_BK = 128;                 // k per stage block (8 x wgmma K = 16)
constexpr int GEMM_WBYTES = GEMM_BN * GEMM_BK * 2;   // 32 KB
constexpr int GEMM_ABYTES = 16 * GEMM_BK * 2;        // 4 KB per 16-token tile
constexpr int GEMM_K8 = GEMM_BK / 8;                 // 16-byte k chunks per stage
constexpr int GEMM_EPI_WARPS = 4;            // the consumer warpgroup: MMA issue and epilogue, thread t = output row t of a tile
constexpr int GEMM_EPI_THREADS = GEMM_EPI_WARPS * 32;
constexpr int GEMM_THREADS = (GEMM_EPI_WARPS + 1) * 32;   // + TMA producer warp
constexpr int GEMM_MAX_SEG = 8;
constexpr int GEMM_STAGE_PITCH = 24;         // halves per row of the A16 epilogue staging buffer (16 tokens + padding, 48 B)
constexpr int GEMM_SMEM_BUDGET = 221184;     // 216 KB for stages (227 KB per block, less the static transpose buffer)
constexpr int GEMM_XPOSE_FLOATS = GEMM_BN * 16;   // accumulator -> row transpose of one 16-token tile (8 KB), shared with the A16 staging
// canonical K-major no-swizzle strides of the two operands in shared memory (wgmma descriptors)
constexpr uint32_t GEMM_W_LBO = 16 * 128;    // weight stage [k8 chunk 16][row group 16][8 rows][16 B]
constexpr uint32_t GEMM_W_SBO = 128;
constexpr uint32_t GEMM_A_LBO = 2 * 128;     // token operand [k8 chunk 16][16 MT rows][16 B]: MT x this (set in the MMA role)
constexpr uint32_t GEMM_A_SBO = 128;

enum OutMode : int {
    OUT_F32 = 0,        // out[m*ldo + n] = y                              (f32 row-major)
    OUT_A16 = 1,        // f16 A16 layout (input of the next projection), optional column groups
    OUT_LERP_A16 = 2,   // v6 ddlerp: f16( xx + sx * (mu[n] + y) ) in A16 layout
};

struct GemmSeg {
    const __half* A;      // A16 activations for this segment (already offset to the segment's first k block)
    int a_k8;             // (unused)
    int KB;               // 128-wide k blocks (K padded up)
    int tiles;            // 128-row output tiles (N padded up)
    int N;                // valid output columns
    int blk_begin;        // first linear stage block of this segment
    int tile_begin;       // first global tile index of this segment
    int out_mode;
    int act;
    const float* bias;    // optional [N], added before the activation
    void* out;
    int ldo;              // OUT_F32: row stride (floats); A16 modes: token rows of the destination (the step's th)
    int grp;              // OUT_A16: columns per destination matrix (0 = single matrix)
    int grp_stride;       // OUT_A16: halves between destination matrices
    const float* aux0;    // OUT_LERP_A16: xx [T, ld_aux]
    const float* aux1;    // OUT_LERP_A16: sx [T, ld_aux]
    const float* aux2;    // OUT_LERP_A16: mu [N]
    int ld_aux;
};

struct GemmParams {
    const uint8_t* W;       // packed stage blocks, linear order
    int nseg;
    int total_blocks;
    int max_contrib;        // workspace slots per tile
    float* ws;              // [total_tiles][max_contrib][128][MT*16] partial tiles
    unsigned* counters;     // [total_tiles], zero between launches
    const int* nrows;       // device: valid token rows
    uint32_t w_lbo, w_sbo, a_lbo, a_sbo;   // wgmma descriptor strides (bytes)
    unsigned long long* trace;             // profiling aid: 8 globaltimer stamps of CTA 0 (null in production)
    GemmSeg seg[GEMM_MAX_SEG];
    // Quantised W' plans (adapter tails, read by the *gemm_tail_kernel instantiations only): each tile of segment s is kbq[s]
    // code blocks, then KB - kbq[s] f16 tail blocks (GEMM_WBYTES each, repack_weight_kernel's layout).  Its code blocks are
    // blocks qblk[s].. of W, its tail blocks blocks tblk[s].. of `tails`, both tile-major.
    const uint8_t* tails;
    const float* scales;                   // FP8: the row scales [global tile][128] behind the code blocks
    int kbq[GEMM_MAX_SEG], qblk[GEMM_MAX_SEG], tblk[GEMM_MAX_SEG];
};

// HALF: ring sized to half an SM's shared memory, so the NEXT projection launch (programmatic
// dependent launch) can be resident and prefetching its first weight blocks while this one drains
// RING 0: as many stages as fit an SM; 1: half of that (two projection CTAs per SM); 2: one stage less than 0, which
// leaves ~40 KB of shared memory so the small kernels around a projection (pre6 / LN / WKV) can share its SMs
template <int MT, int RING = 0>
struct GemmCfg {
    static constexpr int STAGE_BYTES = GEMM_WBYTES + MT * GEMM_ABYTES;
    static constexpr int BUDGET = RING == 1 ? (GEMM_SMEM_BUDGET / 2) : GEMM_SMEM_BUDGET;
    static constexpr int NFIT = (BUDGET / STAGE_BYTES) > 12 ? 12 : (BUDGET / STAGE_BYTES);
    static constexpr int NSTAGE = (RING == 2 && NFIT > 2) ? NFIT - 1 : NFIT;
    static constexpr int BAR_BYTES = 2 * NSTAGE * 8 + 16;
    static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + BAR_BYTES + 64;
};

__device__ __forceinline__ int gemm_find_seg(const GemmParams& p, int b) {
    int s = 0;
#pragma unroll 1
    while (s + 1 < p.nseg && b >= p.seg[s + 1].blk_begin) ++s;
    return s;
}

struct RingPos {
    int stage;
    uint32_t phase;
    template <int NSTAGE>
    __device__ __forceinline__ void advance(int n) {
        stage += n;
        while (stage >= NSTAGE) { stage -= NSTAGE; phase ^= 1u; }
    }
};

// a CTA's block range decomposes into "tile segments": its share of consecutive output tiles
struct SegWalk {
    const GemmParams* p;
    int b, b1, seg, tile_local, kb;
    __device__ __forceinline__ void init(const GemmParams& p_, int b0, int b1_) {
        p = &p_; b = b0; b1 = b1_;
        seg = gemm_find_seg(p_, b0);
        const GemmSeg& sg = p_.seg[seg];
        tile_local = (b0 - sg.blk_begin) / sg.KB;
        kb = (b0 - sg.blk_begin) - tile_local * sg.KB;
    }
    __device__ __forceinline__ bool done() const { return b >= b1; }
    __device__ __forceinline__ int nblk() const { return min(p->seg[seg].KB - kb, b1 - b); }
    __device__ __forceinline__ void next() {
        const GemmSeg& sg = p->seg[seg];
        const int n = nblk();
        b += n;
        kb += n;
        if (kb == sg.KB) {
            kb = 0;
            if (++tile_local == sg.tiles) {
                tile_local = 0;
                if (seg + 1 < p->nseg) ++seg;
            }
        }
    }
};

// ---------------------------------------------------------------------------------------
// Consumer warpgroup: MMAs of a tile segment into register accumulators, then the tile's epilogue.
// ---------------------------------------------------------------------------------------
// element (row r, token column c < 16) of the transpose buffer; the 16-byte column groups are rotated by r / 2 so that
// eight consecutive rows reading the same group hit eight different bank quads
__device__ __forceinline__ int gemm_xpose_index(const int r, const int c) {
    return r * 16 + ((((c >> 2) ^ (r >> 1)) & 3) << 2) + (c & 3);
}
template <int N>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// fragment layout (common.cuh, wgmma) -> thread t holds output row t: v[mt][j] = token 16 mt + j
template <int MT>
__device__ __forceinline__ void gemm_acc_to_rows(float (&acc)[2][8 * MT], float (&v)[MT][16], float* s_x) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
        named_bar_sync(3, GEMM_EPI_THREADS);                  // the previous readers of the buffer are done
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 4; ++e) {                     // fragment pairs 8 mt + 2 e: n8 block e / 2, row half e % 2
                const int i = 8 * mt + 2 * e;
                const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * (e & 1);
                const int c = 8 * (e >> 1) + 2 * (lane & 3);
                *reinterpret_cast<float2*>(s_x + gemm_xpose_index(r, c)) = make_float2(acc[h][i], acc[h][i + 1]);
            }
        named_bar_sync(3, GEMM_EPI_THREADS);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const float4 q = *reinterpret_cast<const float4*>(s_x + gemm_xpose_index(tid, 4 * g));
            v[mt][4 * g] = q.x; v[mt][4 * g + 1] = q.y; v[mt][4 * g + 2] = q.z; v[mt][4 * g + 3] = q.w;
        }
    }
    named_bar_sync(3, GEMM_EPI_THREADS);                      // the buffer is the epilogue's A16 staging next
}

// Epilogue of one tile segment (128 threads, thread t owns output row t of the tile, v = its 16 MT token values):
// deterministic cross-CTA reduction of split tiles, fused epilogue.
// SPLIT (precision 1, MT = 2): the two token tiles are the hi and lo halves of the SAME 16 tokens
// (common.cuh split_h): the accumulator tiles are added before the epilogue and A16 outputs are written as hi / lo again.
template <int MT, bool SPLIT = false>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, const SegWalk& w, const int cta, const int G, float (&v)[MT][16],
                                                   const int nrows, volatile int* s_last_p, __half* s_stage) {
    const int tid = threadIdx.x;
    const unsigned TB = (unsigned)p.total_blocks;
    const GemmSeg& sg = p.seg[w.seg];
    constexpr int ROWF = 16 * MT;
    const unsigned tb0 = (unsigned)(sg.blk_begin + w.tile_local * sg.KB);
    const int c_first = (int)(((unsigned long long)(tb0 + 1) * (unsigned)G - 1) / TB);
    const int c_last = (int)(((unsigned long long)(tb0 + sg.KB) * (unsigned)G - 1) / TB);
    const int ncontrib = c_last - c_first + 1;
    const int gtile = sg.tile_begin + w.tile_local;
    bool do_epilogue = true;
    if (ncontrib > 1) {
        float* wsl = p.ws + ((size_t)gtile * p.max_contrib + (cta - c_first)) * (GEMM_BN * ROWF) + (size_t)tid * ROWF;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int j = 0; j < 16; j += 4)
                *reinterpret_cast<float4*>(wsl + mt * 16 + j) = make_float4(v[mt][j], v[mt][j + 1], v[mt][j + 2], v[mt][j + 3]);
        // publish: the barrier orders every thread's partial stores before thread 0's gpu-scope
        // fence (fences are cumulative), then one counter bump per CTA
        named_bar_sync(3, GEMM_EPI_THREADS);
        if (tid == 0) {
            const unsigned old = atom_add_acq_rel_gpu(p.counters + gtile, 1u);   // release ours, acquire the others'
            *s_last_p = (old == (unsigned)(ncontrib - 1));
            if (*s_last_p) p.counters[gtile] = 0;  // ready for the next launch
        }
        named_bar_sync(3, GEMM_EPI_THREADS);
        do_epilogue = (*s_last_p != 0);
        if (do_epilogue) {
            const float* ws0 = p.ws + (size_t)gtile * p.max_contrib * (GEMM_BN * ROWF) + (size_t)tid * ROWF;
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                for (int j = 0; j < 16; ++j) v[mt][j] = 0.f;
            // fixed slot order -> deterministic; four contributors' loads in flight at a time
            constexpr int UB = (MT >= 4) ? 1 : (MT == 2 ? 2 : 4);
            for (int s0 = 0; s0 < ncontrib; s0 += UB) {
                float4 pv[UB][MT][4];
#pragma unroll
                for (int u = 0; u < UB; ++u) {
                    const float* w_ = ws0 + (size_t)(s0 + u) * (GEMM_BN * ROWF);
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            pv[u][mt][j] = (s0 + u < ncontrib) ? __ldcg(reinterpret_cast<const float4*>(w_ + mt * 16 + 4 * j))
                                                               : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < UB; ++u)
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            v[mt][4 * j] += pv[u][mt][j].x; v[mt][4 * j + 1] += pv[u][mt][j].y;
                            v[mt][4 * j + 2] += pv[u][mt][j].z; v[mt][4 * j + 3] += pv[u][mt][j].w;
                        }
            }
        }
    }
    if (do_epilogue) {
        // The segment descriptor lives in kernel-parameter space (stand-alone kernel) or global
        // memory (whole-step kernel): hoist every field the loop needs into registers once.
        const int n = w.tile_local * GEMM_BN + tid;
        const int segN = sg.N, out_mode = sg.out_mode, act = sg.act, ldo = sg.ldo, grp = sg.grp, grp_stride = sg.grp_stride;
        const int ld_aux = sg.ld_aux;
        void* const outp = sg.out;
        const float* const biasp = sg.bias;
        const float* const aux0 = sg.aux0;
        const float* const aux1 = sg.aux1;
        const float* const aux2 = sg.aux2;
        if (SPLIT) {
            static_assert(!SPLIT || MT == 2, "split operands use two token tiles");
#pragma unroll
            for (int j = 0; j < 16; ++j) v[0][j] += v[MT - 1][j];
        }
        constexpr int MTE = SPLIT ? 1 : MT;        // token tiles the epilogue writes
        const bool row_ok = n < segN;
        const float bias = (row_ok && biasp) ? biasp[n] : 0.f;
        const int mmax = min(nrows, MTE * 16);
        if (out_mode == OUT_F32) {
            if (row_ok) {
                float* o = reinterpret_cast<float*>(outp) + n;
                if (MTE == 1) {         // decode shape: straight from registers, all 16 stores in flight
#pragma unroll
                    for (int m = 0; m < 16; ++m)
                        if (m < mmax) o[(size_t)m * ldo] = apply_act(v[0][m] + bias, act);
                } else {
                    // Multi-tile steps: unrolled over tiles and tokens with compile-time register indices (a dynamically
                    // indexed copy of the accumulator would live in local memory, and next to a 200 KB ring there is no
                    // L1 to hold it); the activation is a compile-time parameter of the unrolled body, otherwise the
                    // run-time switch is replicated 16 MT times and the epilogue outgrows the instruction cache.
                    auto body = [&](auto act_c) {
                        constexpr int ACT_C = decltype(act_c)::value;
#pragma unroll
                        for (int mt = 0; mt < MTE; ++mt)
#pragma unroll
                            for (int j = 0; j < 16; ++j) {
                                const int m = mt * 16 + j;
                                if (m < mmax) o[(size_t)m * ldo] = apply_act(v[mt][j] + bias, ACT_C);
                            }
                    };
                    switch (act) {
                        case ACT_TANH: body(std::integral_constant<int, ACT_TANH>{}); break;
                        case ACT_SIGMOID: body(std::integral_constant<int, ACT_SIGMOID>{}); break;
                        case ACT_SILU: body(std::integral_constant<int, ACT_SILU>{}); break;
                        case ACT_RELU2: body(std::integral_constant<int, ACT_RELU2>{}); break;
                        case ACT_EXPNEGEXP: body(std::integral_constant<int, ACT_EXPNEGEXP>{}); break;
                        case ACT_V7DECAY: body(std::integral_constant<int, ACT_V7DECAY>{}); break;
                        default: body(std::integral_constant<int, ACT_NONE>{}); break;
                    }
                }
            }
        } else {
            // A16 outputs (operand of a following projection).  Thread t holds output row n = one k index of that operand
            // for 16 tokens; the layout wants, per token, 8 consecutive k in one 16-byte chunk.  Written straight from the
            // registers that is one 2-byte store per token and row, four 32-byte sectors per warp instruction -- measured
            // 33 us per 128-token tile (r02_findings.md §8).  So the tile is transposed through 6 KB of shared memory:
            // every thread stages its 16 tokens, then writes two (token, chunk) pairs as 16-byte stores, 16 lanes = 256
            // contiguous bytes.  All 128 epilogue threads take part (rows past the segment stage zeros).
            const bool lerp = (out_mode == OUT_LERP_A16);
            const float mu = (lerp && row_ok) ? aux2[n] : 0.f;
            __half* const base0 = reinterpret_cast<__half*>(outp);
            const int row0 = w.tile_local * GEMM_BN;         // first output row of this tile within the segment
            auto stage_and_store = [&](const int mt, const __half (&h)[16], const int rowoff) {
                uint4 p0, p1;
                p0.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
                p0.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
                p0.z = (uint32_t)__half_as_ushort(h[4]) | ((uint32_t)__half_as_ushort(h[5]) << 16);
                p0.w = (uint32_t)__half_as_ushort(h[6]) | ((uint32_t)__half_as_ushort(h[7]) << 16);
                p1.x = (uint32_t)__half_as_ushort(h[8]) | ((uint32_t)__half_as_ushort(h[9]) << 16);
                p1.y = (uint32_t)__half_as_ushort(h[10]) | ((uint32_t)__half_as_ushort(h[11]) << 16);
                p1.z = (uint32_t)__half_as_ushort(h[12]) | ((uint32_t)__half_as_ushort(h[13]) << 16);
                p1.w = (uint32_t)__half_as_ushort(h[14]) | ((uint32_t)__half_as_ushort(h[15]) << 16);
                *reinterpret_cast<uint4*>(s_stage + tid * GEMM_STAGE_PITCH) = p0;
                *reinterpret_cast<uint4*>(s_stage + tid * GEMM_STAGE_PITCH + 8) = p1;
                named_bar_sync(3, GEMM_EPI_THREADS);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int q = tid + GEMM_EPI_THREADS * i;
                    const int c = q >> 4, m = q & 15;               // chunk of 8 rows, token of the tile
                    const int nc = row0 + c * 8;                    // first output row of the chunk (N % 8 == 0: whole chunks)
                    if (nc < segN && mt * 16 + m < mmax) {
                        const __half* src = s_stage + (c * 8) * GEMM_STAGE_PITCH + m;
                        uint4 o;
                        o.x = (uint32_t)__half_as_ushort(src[0]) | ((uint32_t)__half_as_ushort(src[GEMM_STAGE_PITCH]) << 16);
                        o.y = (uint32_t)__half_as_ushort(src[2 * GEMM_STAGE_PITCH]) | ((uint32_t)__half_as_ushort(src[3 * GEMM_STAGE_PITCH]) << 16);
                        o.z = (uint32_t)__half_as_ushort(src[4 * GEMM_STAGE_PITCH]) | ((uint32_t)__half_as_ushort(src[5 * GEMM_STAGE_PITCH]) << 16);
                        o.w = (uint32_t)__half_as_ushort(src[6 * GEMM_STAGE_PITCH]) | ((uint32_t)__half_as_ushort(src[7 * GEMM_STAGE_PITCH]) << 16);
                        __half* base = base0;
                        int nn = nc;
                        if (grp > 0) {
                            const int gi = nc / grp;
                            base += (size_t)gi * grp_stride;
                            nn = nc - gi * grp;
                        }
                        *reinterpret_cast<uint4*>(base + a16_index(mt * 16 + m + rowoff, nn, ldo)) = o;
                    }
                }
                named_bar_sync(3, GEMM_EPI_THREADS);            // the staging buffer is rewritten by the next tile
            };
            auto body = [&](auto act_c) {
                constexpr int ACT_C = decltype(act_c)::value;
#pragma unroll
                for (int mt = 0; mt < MTE; ++mt) {
                    if (mt * 16 < mmax) {                           // uniform over the CTA
                        float x0[16], x1[16];                       // the lerp operands of the tile's 16 tokens, requested together
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int m = mt * 16 + j;
                            const bool ok = lerp && row_ok && m < mmax;
                            const size_t a_ = (size_t)m * ld_aux + n;
                            x0[j] = ok ? aux0[a_] : 0.f;
                            x1[j] = ok ? aux1[a_] : 0.f;
                        }
                        __half hi[16], lo[16];
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            float y = apply_act(v[mt][j] + bias, ACT_C);
                            if (lerp) y = x0[j] + x1[j] * (mu + y);
                            if (!row_ok) y = 0.f;
                            if (SPLIT) split_h(y, hi[j], lo[j]);
                            else hi[j] = f2h_sat(y);
                        }
                        stage_and_store(mt, hi, 0);
                        if (SPLIT) stage_and_store(mt, lo, 16);
                    }
                }
            };
            switch (act) {
                case ACT_TANH: body(std::integral_constant<int, ACT_TANH>{}); break;
                case ACT_SIGMOID: body(std::integral_constant<int, ACT_SIGMOID>{}); break;
                case ACT_SILU: body(std::integral_constant<int, ACT_SILU>{}); break;
                case ACT_RELU2: body(std::integral_constant<int, ACT_RELU2>{}); break;
                case ACT_EXPNEGEXP: body(std::integral_constant<int, ACT_EXPNEGEXP>{}); break;
                case ACT_V7DECAY: body(std::integral_constant<int, ACT_V7DECAY>{}); break;
                default: body(std::integral_constant<int, ACT_NONE>{}); break;
            }
        }
    }
}

template <int MT, int NSTAGE, int STAGE_BYTES, bool SPLIT>
__device__ __forceinline__ void gemm_consumer_role(const GemmParams& p, const int cta, const int G, const int b0, const int b1,
                                                   const uint32_t smem_base, const uint32_t full_bar, const uint32_t empty_bar,
                                                   const int nrows, volatile int* s_last_p, float* s_x, unsigned long long* tr) {
    const int lane = threadIdx.x & 31;
    const uint32_t w_lbo = p.w_lbo, w_sbo = p.w_sbo, a_sbo = p.a_sbo;
    constexpr uint32_t a_lbo = 16 * MT * 16;          // bytes between the k8 chunks of the token operand: 16 MT rows x 16 B
    RingPos rp{0, 0u};
    SegWalk w;
    w.init(p, b0, b1);
    while (!w.done()) {
        const int nblk = w.nblk();
        float acc[2][8 * MT];                          // weight rows 0-63 and 64-127 of the tile
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 8 * MT; ++i) acc[h][i] = 0.f;
        int prev = -1;
        for (int i = 0; i < nblk; ++i) {
            mbar_wait(full_bar + rp.stage * 8, rp.phase, 12);
            if (tr && threadIdx.x == 0 && i == 0 && rp.stage == 0 && rp.phase == 0) tr[3] = globaltimer_ns();
            const uint32_t st = smem_base + rp.stage * STAGE_BYTES;
            wgmma_fence_operand(acc[0]);
            wgmma_fence_operand(acc[1]);
            wgmma_fence();
            // one MMA per k16 step and weight half over all 16 x MT token rows of the stage (N = 16 MT): the token operand
            // of a stage is one canonical tile [k8 chunk][16 MT rows][16 B] (common.cuh), chunk stride = 16 MT x 16 bytes
#pragma unroll
            for (int k16 = 0; k16 < GEMM_BK / 16; ++k16) {
                const uint64_t bdesc = gmma_desc(st + GEMM_WBYTES + k16 * 2 * a_lbo, a_lbo, a_sbo);
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    wgmma_f16<16 * MT>(acc[h], gmma_desc(st + h * 8 * w_sbo + k16 * 2 * w_lbo, w_lbo, w_sbo), bdesc);
            }
            wgmma_commit();
            wgmma_wait<1>();                           // the previous stage's MMAs have retired: its slot may be refilled
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar + prev * 8);
            }
            prev = rp.stage;
            rp.advance<NSTAGE>(1);
        }
        wgmma_wait<0>();
        wgmma_fence_operand(acc[0]);
        wgmma_fence_operand(acc[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + prev * 8);
        float v[MT][16];
        gemm_acc_to_rows<MT>(acc, v, s_x);
        gemm_epilogue_tile<MT, SPLIT>(p, w, cta, G, v, nrows, s_last_p, reinterpret_cast<__half*>(s_x));
        w.next();
    }
    if (tr && threadIdx.x == 0) tr[4] = globaltimer_ns();
}

// ---------------------------------------------------------------------------------------
// stand-alone kernel: warps 0-3 consumer warpgroup (MMA + epilogue), warp 4 TMA producer
// ---------------------------------------------------------------------------------------
template <int MT, int RING = 0, bool SPLIT = false>
__global__ void __launch_bounds__(GEMM_THREADS, RING == 1 ? 2 : 1) gemm_kernel(const __grid_constant__ GemmParams p) {
    using Cfg = GemmCfg<MT, RING>;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int s_last;
    __shared__ __align__(16) float s_x[GEMM_XPOSE_FLOATS];     // accumulator transpose, then A16 epilogue staging
    static_assert(GEMM_EPI_THREADS * GEMM_STAGE_PITCH * 2 <= GEMM_XPOSE_FLOATS * 4, "A16 staging fits the transpose buffer");
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t full_bar = smem_base + Cfg::NSTAGE * Cfg::STAGE_BYTES;
    const uint32_t empty_bar = full_bar + Cfg::NSTAGE * 8;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long TB = p.total_blocks;
    const int G = gridDim.x, cta = blockIdx.x;
    const int b0 = (int)((long long)cta * TB / G);
    const int b1 = (int)((long long)(cta + 1) * TB / G);
    unsigned long long* const tr = (p.trace && cta == 0) ? p.trace : nullptr;
    auto stamp = [&](int i) {
        if (tr) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
            tr[i] = t;
        }
    };

    if (tid == 0) {
        stamp(0);
        for (int s = 0; s < Cfg::NSTAGE; ++s) {
            mbar_init(full_bar + s * 8, 1);
            mbar_init(empty_bar + s * 8, GEMM_EPI_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) stamp(1);
    pdl_launch_dependents();     // let the next kernel's CTAs queue up and prefetch their weights

    if (warp == GEMM_EPI_WARPS) {
        // ===================== producer: one lane streams stage blocks =====================
        if (lane == 0) {
            const uint64_t pol_w = l2_policy_evict_first();
            const uint64_t pol_a = l2_policy_evict_last();
            // Weights never change: the first ring-full of weight blocks is requested BEFORE
            // waiting on the preceding kernel (programmatic dependent launch), so HBM keeps
            // streaming across the kernel boundary.  Activations are fetched after the wait.
            const int npre = min(b1 - b0, Cfg::NSTAGE);
            for (int i = 0; i < npre; ++i) {
                const uint32_t st = smem_base + i * Cfg::STAGE_BYTES;
                mbar_expect_tx(full_bar + i * 8, Cfg::STAGE_BYTES);
                bulk_g2s_hint(st, p.W + (size_t)(b0 + i) * GEMM_WBYTES, GEMM_WBYTES, full_bar + i * 8, pol_w);
            }
            pdl_wait();
            stamp(2);
            int seg = gemm_find_seg(p, b0);
            const GemmSeg* sg = &p.seg[seg];
            int kb = (b0 - sg->blk_begin) % sg->KB;
            int blocks_left_in_seg = sg->blk_begin + sg->tiles * sg->KB - b0;
            int stage = 0;
            uint32_t ephase = 1;            // parity of the "previous" phase of the empty barriers
            for (int b = b0, it = 0; b < b1; ++b, ++it) {
                const uint32_t st = smem_base + stage * Cfg::STAGE_BYTES;
                const uint32_t fb = full_bar + stage * 8;
                if (it >= Cfg::NSTAGE) {
                    mbar_wait(empty_bar + stage * 8, ephase, 14);
                    mbar_expect_tx(fb, Cfg::STAGE_BYTES);
                    bulk_g2s_hint(st, p.W + (size_t)b * GEMM_WBYTES, GEMM_WBYTES, fb, pol_w);
                }
                // the k block's slice of all MT token tiles is one contiguous run of the A16 layout (common.cuh)
                bulk_g2s_hint(st + GEMM_WBYTES, sg->A + (size_t)kb * A16_KB_HALVES, MT * GEMM_ABYTES, fb, pol_a);
                if (++stage == Cfg::NSTAGE) { stage = 0; ephase ^= 1; }
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
        // ===================== consumer warpgroup: MMA + epilogue =====================
        pdl_wait();
        if (tid == 0) stamp(5);
        gemm_consumer_role<MT, Cfg::NSTAGE, Cfg::STAGE_BYTES, SPLIT>(p, cta, G, b0, b1, smem_base, full_bar, empty_bar, *p.nrows, &s_last,
                                                                     s_x, tr);
        if (tid == 0) stamp(6);
        if (tid == 0 && p.trace) {       // every CTA: SM id and the time its MMAs were done (skew across the grid)
            unsigned smid;
            asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
            p.trace[8 + 3 * cta] = smid;
            p.trace[8 + 3 * cta + 1] = globaltimer_ns();
        }
    }
    __syncthreads();
    if (tid == 0) stamp(7);
    if (tid == 0 && p.trace) p.trace[8 + 3 * cta + 2] = globaltimer_ns();
}

// ---------------------------------------------------------------------------------------
// One-time weight re-tiling:  W[N, K] row-major f16  ->  stage blocks in the canonical
// K-major / no-swizzle layout:  block(tile, kb) = [k8 chunk 16][row group 16][row 8][8 halves], zero padded.
// Supports a row-parallel / column-parallel shard: source sub-matrix rows [n0, n0+N), cols [k0, k0+K)
// of a matrix with row stride ld.  Block (tile, kb) goes to block tile * dst_kb + kb of dst (dst_kb >= KB: the first KB blocks
// of every tile row of a wider plan, whose other blocks are left as they are).
// ---------------------------------------------------------------------------------------
__global__ void repack_weight_kernel(const __half* __restrict__ src, int ld, int n0, int k0, int N, int K,
                                     int tiles, int KB, int dst_kb, uint4* __restrict__ dst) {
    // one thread per 16-byte chunk (8 halves)
    const size_t nchunk = (size_t)tiles * KB * (GEMM_WBYTES / 16);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nchunk; i += (size_t)gridDim.x * blockDim.x) {
        size_t r = i;
        const int row = r % 8; r /= 8;       // row inside the 8-row core matrix
        const int mi = r % 16; r /= 16;      // row group
        const int kj = r % GEMM_K8; r /= GEMM_K8;   // 8-half (16-byte) k chunk
        const int kb = r % KB; r /= KB;
        const int tile = (int)r;
        const int n = tile * GEMM_BN + mi * 8 + row;
        const int k = kb * GEMM_BK + kj * 8;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (n < N) {
            const __half* s = src + (size_t)(n0 + n) * ld + k0 + k;
            if (k + 8 <= K && ((reinterpret_cast<uintptr_t>(s) & 15) == 0)) {
                v = *reinterpret_cast<const uint4*>(s);
            } else {
                __half tmp[8];
                for (int e = 0; e < 8; ++e) tmp[e] = (k + e < K) ? s[e] : __float2half(0.f);
                v = *reinterpret_cast<uint4*>(tmp);
            }
        }
        dst[((size_t)tile * dst_kb + kb) * (GEMM_WBYTES / 16) + i % (GEMM_WBYTES / 16)] = v;
    }
}

// The inverse of repack_weight_kernel for a whole matrix (n0 = k0 = 0, dst_kb = KB, K a multiple of 8): the stage blocks
// back into dense [N][K] f16 rows, padding dropped.  The quantised head (b200rwkv_head_format) is quantised from these rows.
__global__ void unpack_weight_kernel(const uint4* __restrict__ src, int N, int K, int tiles, int KB, __half* __restrict__ dst) {
    const size_t nchunk = (size_t)tiles * KB * (GEMM_WBYTES / 16);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nchunk; i += (size_t)gridDim.x * blockDim.x) {
        size_t r = i;
        const int row = r % 8; r /= 8;
        const int mi = r % 16; r /= 16;
        const int kj = r % GEMM_K8; r /= GEMM_K8;
        const int kb = r % KB; r /= KB;
        const int n = (int)r * GEMM_BN + mi * 8 + row;
        const int k = kb * GEMM_BK + kj * 8;
        if (n < N && k < K) *reinterpret_cast<uint4*>(dst + (size_t)n * K + k) = src[i];
    }
}

}  // namespace b200
