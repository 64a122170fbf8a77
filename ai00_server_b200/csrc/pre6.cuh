// Decode-shaped (<= 16 tokens) front half of a time-mix / channel-mix block as ONE launch of 16 clusters x 8 CTAs.
//
// Replaces, on the path `Runtime::infer` (reference run.rs:1143; SURVEY.md §2.2 K1-K3, App. A), web-rwkv's
// `layer_norm` + `token_shift` (+ for RWKV-6 the two LoRA matmuls of the data-dependent token shift) dispatches.
//
// Why: as separate launches, the one-CTA-per-token LN launch and the two 2.6 MB LoRA GEMM launches of every RWKV-6 layer
// are time in which HBM idles, comparable to the layer's weight streaming.  Nothing here is bandwidth: it is a chain of L2 round trips, so the shape is chosen for
// the shortest chain:
//   phase 1  cluster g = token g, CTA rank s = channel slice s (C/8 channels, one float4 per thread): residual update, LN
//            statistics through distributed shared memory (two cluster syncs), token shift, static mixes.
//   -- grid barrier (RWKV-6 only) --
//   phase 2  cluster g = 1/16 of the 5*Dm LoRA rows, rank s = K slice s: tokens are the M=16 side of `mma.sync.m16n8k16`,
//            W1 fragments were loaded straight from the row-major weight BEFORE griddepcontrol.wait; warps split K, the
//            cluster reduces the 8 K slices through DSMEM in a fixed order, tanh, f16.
//   -- grid barrier --
//   phase 3  CTA b = channels [32 b, 32 b + 32) x 5 mixes: W2 fragments (also preloaded), y = xx + sx * (mu + W2 tanh),
//            written as the A16 operands of the R/K/V/G/decay projections.
// The tensor cores are used through legacy mma.sync on purpose: each CTA issues a few dozen MMAs, and wgmma would add
// warpgroup-wide issue plus shared-memory operand staging to a chain that is pure latency.
// The kernel keeps < 16 KB of shared memory so the next projection's CTAs (200 KB ring, launched early through PDL) can
// sit on the same SMs and fill their rings while these phases run.
#pragma once
#include <cooperative_groups.h>

#include "mix.cuh"

namespace b200 {
namespace cg = cooperative_groups;

constexpr int PRE_CLUSTER = 8;        // CTAs per cluster (portable maximum)
constexpr int PRE_NCLUSTER = 16;      // = tokens of a decode-shaped step
constexpr int PRE_GRID = PRE_CLUSTER * PRE_NCLUSTER;
constexpr int PRE_THREADS = 256;
constexpr int PRE_MAX_C = 4096;
constexpr int PRE_NT2 = 3;            // n-tiles (8 LoRA rows each) per cluster in phase 2
constexpr int PRE_KSW = 4;            // k-steps (16 wide) per warp in phase 2
constexpr int PRE_TILES3 = 3;         // n-tiles (8 channels x one mix) per warp in phase 3

struct Pre6Params {
    LnMixParams ln;           // phase 1 (RWKV-6: n_mix = 1 -> xxx; xx_out / sx_out feed phase 3)
    const __half* W1;         // [5*Dm][C] row-major (time_mix_w1 as stored in the .st)
    const __half* W2;         // [5][C][Dm]        (time_mix_w2)
    const float* mu[5];       // time_mix_{w,k,v,r,g}
    __half* lora;             // five A16 [16][Dm] matrices: tanh(W1 xxx)
    int lora_stride;          // halves between them
    int lora_kq;              // (unused: the token-row count of the A16 operands is 16, or 32 with split operands)
    __half* out[5];           // A16 [16][C] operands of decay-LoRA, K, V, R, G
    int Dm;
    unsigned* gbar;           // two arrival counters, 128 bytes apart
};

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t b0, const uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Grid barrier of the 16 clusters: hardware cluster barrier, one fire-and-forget arrival per cluster on `mine`, spin
// until all 16 arrived, cluster barrier again.  The two barriers of a launch use two counters and CTA 0 re-arms them
// where no arrival can race with the reset:
//   `reset_before` (barrier 1 re-arms counter 2): its last use was the previous launch, and the store is ordered
//       before CTA 0's own release-arrival, which every cluster acquires before it can reach barrier 2;
//   `reset_after`  (barrier 2 re-arms counter 1): everybody arrived at barrier 2, so nobody still polls counter 1, and
//       its next arrivals belong to the next launch.
__device__ __forceinline__ void pre_grid_barrier(cg::cluster_group& cl, const unsigned rank, unsigned* mine, unsigned* reset_before,
                                                 unsigned* reset_after, const unsigned tag) {
    cl.sync();
    if (rank == 0 && threadIdx.x == 0) {
        if (blockIdx.x == 0 && reset_before) st_relaxed_gpu(reset_before, 0u);
        red_add_release_gpu(mine, 1u);
        SpinGuard sg_;
        unsigned seen;
        while ((seen = ld_acquire_gpu(mine)) < (unsigned)PRE_NCLUSTER) sg_.poll(WD_GRIDBAR, 0x600u + tag, seen, blockIdx.x);
        if (blockIdx.x == 0 && reset_after) st_relaxed_gpu(reset_after, 0u);
        __threadfence();
    }
    cl.sync();
}

// sum over the cluster of a value every thread of the CTA already holds; `xch` must be a buffer no earlier exchange of
// this launch used (a fast CTA may write the next exchange while a slow one still reads this one)
__device__ __forceinline__ float cluster_sum(cg::cluster_group& cl, const unsigned rank, float* xch, const float v) {
    if (threadIdx.x < PRE_CLUSTER) cl.map_shared_rank(xch, threadIdx.x)[rank] = v;
    cl.sync();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PRE_CLUSTER; ++i) s += xch[i];      // fixed order: identical in all CTAs
    return s;
}

// one float4 of the updated residual; same arithmetic as residual_row()
__device__ __forceinline__ float4 residual_vec(const ResidualSrc& r, const int t, const int c) {
    const size_t base = (size_t)t * r.C + c;
    float4 a = ld4(r.x_in + base);
    if (r.n_parts == 0) return a;
    float4 v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = (q < r.n_parts) ? ld4(r.parts[q] + base) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 gt = make_float4(1.f, 1.f, 1.f, 1.f);
    if (r.n_gate > 0) {
        const int gb = c / r.gate_cl;
        const float* gp = r.gates[0];       // selected without a dynamic index: keeps the struct in registers
#pragma unroll
        for (int i = 1; i < 8; ++i) gp = (gb == i) ? r.gates[i] : gp;
        gt = ld4(gp + (size_t)t * r.gate_cl + (c - gb * r.gate_cl));
    }
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < 8; ++q) add4(s, v[q]);
    if (r.n_gate > 0) { s.x *= gt.x; s.y *= gt.y; s.z *= gt.z; s.w *= gt.w; }
    add4(a, s);
    return a;
}

// LN statistics of a row spread over the cluster: each CTA reduces its slice to (mean_i, M2_i) and ONE exchange through
// distributed shared memory combines them (Chan et al.): mean = avg mean_i, M2 = sum M2_i + n_i sum (mean_i - mean)^2.
// `xch` must be a buffer no earlier exchange of this launch used (a fast CTA may write the next exchange while a slow
// one still reads this one).
__device__ __forceinline__ void slice_stats(cg::cluster_group& cl, const unsigned rank, const int C, const bool act, const float4 a,
                                            float* red, float* xch, float& mean, float& rstd) {
    const int Cs = C / PRE_CLUSTER;
    const float s = act ? (a.x + a.y) + (a.z + a.w) : 0.f;
    const float mi = block_sum(s, red) / (float)Cs;
    float s2 = 0.f;
    if (act) {
        const float dx = a.x - mi, dy = a.y - mi, dz = a.z - mi, dw = a.w - mi;
        s2 = (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float m2i = block_sum(s2, red);
    if (threadIdx.x < PRE_CLUSTER) {
        float* dst = cl.map_shared_rank(xch, threadIdx.x);
        dst[rank] = mi;
        dst[PRE_CLUSTER + rank] = m2i;
    }
    cl.sync();
    float ms = 0.f;
#pragma unroll
    for (int i = 0; i < PRE_CLUSTER; ++i) ms += xch[i];      // fixed order: identical in all CTAs
    mean = ms / (float)PRE_CLUSTER;
    float m2 = 0.f;
#pragma unroll
    for (int i = 0; i < PRE_CLUSTER; ++i) {
        const float d = xch[i] - mean;
        m2 += xch[PRE_CLUSTER + i] + (float)Cs * d * d;
    }
    rstd = 1.0f / sqrtf(m2 / (float)C + LN_EPS);
}

template <int NMIX>
struct PreLnStatic {       // operands of phase 1 that no kernel of this step writes: requested before griddepcontrol.wait
    float4 w, b;
    float4 mu[NMIX];
    int T, slot, prev_t, last;     // step metadata is uploaded before the step's first launch
    float* hid;                    // hidden-row buffer of this stage (LnMixParams::hid_slot) or null
    float* snap;                   // snapshot record of this token (LnMixParams::snap_rec) or null
};

template <int NMIX>
__device__ __forceinline__ PreLnStatic<NMIX> pre_ln_static(const LnMixParams& p, const int t, const unsigned rank) {
    const int Cs = p.C / PRE_CLUSTER;
    PreLnStatic<NMIX> st;
    st.T = p.meta.T();
    st.slot = p.meta.tok_slot()[t];
    st.prev_t = p.meta.tok_prev()[t];
    st.last = p.meta.tok_last()[t];
    st.hid = p.hid_slot ? *p.hid_slot : nullptr;
    st.snap = (p.snap_rec && p.commit_dst && t < st.T) ? p.snap_rec[t] : nullptr;
    const bool act = 4 * (int)threadIdx.x < Cs;
    const int c = act ? (int)rank * Cs + 4 * (int)threadIdx.x : 0;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    st.w = act ? ld4(p.ln_w + c) : z4;
    st.b = act ? ld4(p.ln_b + c) : z4;
#pragma unroll
    for (int m = 0; m < NMIX; ++m) st.mu[m] = (act && m < p.n_mix) ? ld4(p.mu[m] + c) : z4;
    return st;
}

// phase 1 for token t, channel slice `rank` (thread owns channels rank*C/8 + 4*tid .. +3)
// WIDE: a step of up to 128 tokens (the batch-invariant mode), whose A16 operands hold p.kq_tile token rows; a token's
// arithmetic is the decode step's
template <int NMIX, bool SPLIT = false, bool WIDE = false>
__device__ __forceinline__ void pre_ln_slice(const LnMixParams& p, const int t, cg::cluster_group& cl, const unsigned rank,
                                             const PreLnStatic<NMIX>& st, float* red, float (*xch)[2 * PRE_CLUSTER]) {
    const int C = p.C, Cs = C / PRE_CLUSTER;
    const bool act = 4 * (int)threadIdx.x < Cs;
    const int c = act ? (int)rank * Cs + 4 * (int)threadIdx.x : 0;
    const int slot = st.slot, prev_t = st.prev_t;
    const bool last = st.last != 0;
    const ResidualSrc r = make_residual_src(p);
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    // one batch of loads: residual operands, shift state, the row this stage commits
    float4 pv = z4, cm = z4;
    if (act && prev_t < 0) pv = ld4(p.shift_state + (size_t)slot * C + c);
    const bool commit = act && last && p.commit_dst;
    const bool snap = act && st.snap;
    if (commit || snap) cm = ld4(p.commit_src + (size_t)t * C + c);
    float4 a = act ? residual_vec(r, t, c) : z4;
    if (act && (p.x_out != p.x_in || p.n_parts > 0)) *reinterpret_cast<float4*>(p.x_out + (size_t)t * C + c) = a;
    if (act && st.hid) *reinterpret_cast<float4*>(st.hid + (size_t)t * C + c) = a;
    float mean, rstd;
    slice_stats(cl, rank, C, act, a, red, xch[0], mean, rstd);
    if (prev_t >= 0) {          // multi-token slot: previous token's LN output, recomputed (uniform over the cluster)
        float pmean, prstd;
        pv = act ? residual_vec(r, prev_t, c) : z4;
        slice_stats(cl, rank, C, act, pv, red, xch[1], pmean, prstd);
        pv = ln_apply(pv, pmean, prstd, st.w, st.b);
    }
    if (!act) return;
    a = ln_apply(a, mean, rstd, st.w, st.b);          // xx
    float4 sx;
    sx.x = pv.x - a.x; sx.y = pv.y - a.y; sx.z = pv.z - a.z; sx.w = pv.w - a.w;
    *reinterpret_cast<float4*>(p.xx_out + (size_t)t * C + c) = a;
    if (p.sx_out) *reinterpret_cast<float4*>(p.sx_out + (size_t)t * C + c) = sx;
    if (commit) *reinterpret_cast<float4*>(p.commit_dst + (size_t)slot * C + c) = cm;
    if (snap) *reinterpret_cast<float4*>(st.snap + p.snap_off + c) = cm;
#pragma unroll
    for (int m = 0; m < NMIX; ++m) {
        if (m < p.n_mix) {
            const float4 mu = st.mu[m];
            if (SPLIT) {
                uint2 hi, lo;
                split_pack_h2(a.x + sx.x * mu.x, a.y + sx.y * mu.y, hi.x, lo.x);
                split_pack_h2(a.z + sx.z * mu.z, a.w + sx.w * mu.w, hi.y, lo.y);
                *reinterpret_cast<uint2*>(p.mix_out[m] + a16_index(t, c, 32)) = hi;
                *reinterpret_cast<uint2*>(p.mix_out[m] + a16_index(t + 16, c, 32)) = lo;
            } else {
                uint2 o;
                o.x = pack_h2(a.x + sx.x * mu.x, a.y + sx.y * mu.y);
                o.y = pack_h2(a.z + sx.z * mu.z, a.w + sx.w * mu.w);
                *reinterpret_cast<uint2*>(p.mix_out[m] + a16_index(t, c, WIDE ? p.kq_tile : 16)) = o;
            }
        }
    }
}

// LN stage alone (channel mix of every version, time mix of RWKV-5/7): 16 clusters x 8, no grid barrier.  WIDE (the
// batch-invariant mode's steps of 17..128 tokens, never split): one cluster per token row of the step, so every row is
// reduced in the decode step's order.
template <bool SPLIT = false, bool WIDE = false>
__global__ void __launch_bounds__(PRE_THREADS) ln_mix_cluster_kernel(const __grid_constant__ LnMixParams p) {
    static_assert(!(SPLIT && WIDE), "split operands run decode-shaped steps only");
    __shared__ float red[32];
    __shared__ float xch[2][2 * PRE_CLUSTER];
    cg::cluster_group cl = cg::this_cluster();
    const unsigned rank = cl.block_rank();
    const int t = blockIdx.x / PRE_CLUSTER;
    trace_stamp(p.trace, 0);
    pdl_launch_dependents();
    const PreLnStatic<6> st = pre_ln_static<6>(p, t, rank);
    cl.sync();       // every CTA of the cluster is executing before anyone writes into a peer's shared memory (off the critical path)
    pdl_wait();
    trace_stamp(p.trace, 1);
    if (t >= st.T) return;                // uniform over the cluster
    pre_ln_slice<6, SPLIT, WIDE>(p, t, cl, rank, st, red, xch);
    cl.sync();                            // no CTA leaves while a peer may still write into its exchange buffers
    trace_stamp(p.trace, 7);
}

// KD = Dm / 16.  WIDE: phases 2 and 3 of a step of 17..128 tokens (the batch-invariant mode; the wide ln_mix_cluster_kernel
// launch before it ran phase 1 for every token): the same 16 x 8 grid walks the step's token groups of 16, so each token
// meets the same W1 / W2 fragments, K slices and reduction order as in a decode step.  Barrier 1 stays to keep the counter
// protocol of pre_grid_barrier.
template <int KD, bool SPLIT = false, bool WIDE = false>
__global__ void __launch_bounds__(PRE_THREADS, 2) pre6_kernel(const __grid_constant__ Pre6Params p) {
    static_assert(!(SPLIT && WIDE), "split operands run decode-shaped steps only");
    __shared__ float red[32];
    __shared__ float xch[2][2 * PRE_CLUSTER];
    __shared__ __align__(16) float red2[8][PRE_NT2 * 4 * 32];
    __shared__ float part[PRE_NT2 * 4 * 32];
    cg::cluster_group cl = cg::this_cluster();
    const unsigned rank = cl.block_rank();
    const int g = blockIdx.x / PRE_CLUSTER;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, grp = lane >> 2, tig = lane & 3;
    constexpr int Dm = KD * 16;
    const int TH = WIDE ? p.ln.kq_tile : (SPLIT ? 32 : 16);     // token rows of the A16 operands (16 / 32 in a decode-shaped step)
    constexpr int NR = 5 * Dm;                                  // LoRA rows
    constexpr int RG = (NR + PRE_NCLUSTER - 1) / PRE_NCLUSTER;  // rows per cluster (10 / 20)
    static_assert(RG <= PRE_NT2 * 8, "row group does not fit the n-tiles");
    const int C = p.ln.C, Cs = C / PRE_CLUSTER;
    unsigned long long* const tr = p.ln.trace;
    trace_stamp(tr, 0);
    auto cta_stamp = [&](int i) {       // profiling aid: every CTA's {entry, wait released, phase 1 done} for skew analysis
        if (tr && threadIdx.x == 0) tr[8 + 3 * blockIdx.x + i] = globaltimer_ns();
    };
    cta_stamp(0);
    pdl_launch_dependents();

    // ---------------- static operands (weights): in flight while the previous kernel drains ----------------
    const PreLnStatic<1> st = pre_ln_static<1>(p.ln, g, rank);
    // phase 2: B fragments of W1, rows g*RG + nt*8 + grp, k = rank*Cs + kstep*16 + tig*2 (+8)
    uint32_t w1f[PRE_KSW][PRE_NT2][2];
    const int ksteps = Cs / 16;
#pragma unroll
    for (int i = 0; i < PRE_KSW; ++i) {
        const int kstep = warp + 8 * i;
        const int kb = (int)rank * Cs + kstep * 16 + tig * 2;
#pragma unroll
        for (int nt = 0; nt < PRE_NT2; ++nt) {
            const int nrow = nt * 8 + grp, n = g * RG + nrow;
            const bool ok = kstep < ksteps && nrow < RG && n < NR;
            const __half* src = p.W1 + (size_t)n * C + kb;
            w1f[i][nt][0] = ok ? *reinterpret_cast<const uint32_t*>(src) : 0u;
            w1f[i][nt][1] = ok ? *reinterpret_cast<const uint32_t*>(src + 8) : 0u;
        }
    }
    // phase 3: this CTA's chunks (8 channels each) x 5 mixes; warp takes tiles warp, warp+8, warp+16
    const int nchunks = C / 8;
    const int cpc = (nchunks + PRE_GRID - 1) / PRE_GRID;
    const int ch_lo = min((int)blockIdx.x * cpc, nchunks), ch_hi = min(ch_lo + cpc, nchunks);
    const int nch = ch_hi - ch_lo, ntiles = nch * 5;
    uint32_t w2f[PRE_TILES3][KD][2];
    float2 mu3[PRE_TILES3];
    int tj[PRE_TILES3], tc0[PRE_TILES3];
#pragma unroll
    for (int i = 0; i < PRE_TILES3; ++i) {
        const int q = warp + 8 * i;
        const bool ok = q < ntiles;
        const int j = ok ? q / nch : 0, ci = ok ? q - j * nch : 0;
        tj[i] = ok ? j : -1;
        tc0[i] = (ch_lo + ci) * 8;
        const __half* src = p.W2 + ((size_t)j * C + tc0[i] + grp) * Dm + tig * 2;
#pragma unroll
        for (int ks = 0; ks < KD; ++ks) {
            w2f[i][ks][0] = ok ? *reinterpret_cast<const uint32_t*>(src + ks * 16) : 0u;
            w2f[i][ks][1] = ok ? *reinterpret_cast<const uint32_t*>(src + ks * 16 + 8) : 0u;
        }
        mu3[i] = ok ? *reinterpret_cast<const float2*>(p.mu[j] + tc0[i] + tig * 2) : make_float2(0.f, 0.f);
    }
    cl.sync();       // every CTA of the cluster is executing before anyone writes into a peer's shared memory (off the critical path)
    pdl_wait();
    trace_stamp(tr, 1);
    cta_stamp(1);
    const int T = WIDE ? st.T : min(st.T, 16);
    const int ngrp = WIDE ? (T + 15) / 16 : 1;                  // token groups of 16

    // ---------------- phase 1: token g ----------------
    if (!WIDE && g < T) pre_ln_slice<1, SPLIT>(p.ln, g, cl, rank, st, red, xch);
    trace_stamp(tr, 2);
    cta_stamp(2);
    pre_grid_barrier(cl, rank, p.gbar, p.gbar + 32, nullptr, 1);
    trace_stamp(tr, 3);

    // ---------------- phase 2: tanh(W1 xxx), rows of cluster g, K slice `rank` ----------------
    for (int q = 0; q < ngrp; ++q) {
        if (q > 0) cl.sync();        // every peer has read `part` of the previous group before it is rewritten
        const int t0 = 16 * q;
        float acc[PRE_NT2][4];
#pragma unroll
        for (int nt = 0; nt < PRE_NT2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
        // split operands: the lo halves of the 16 tokens are the second 16-token tile of the same A16 buffer
#pragma unroll
        for (int sp = 0; sp < (SPLIT ? 2 : 1); ++sp) {
            const __half* xa = p.ln.mix_out[0];      // A16: token tile 0 (hi) / 1 (lo) of every k block
            uint32_t af[PRE_KSW][4];
#pragma unroll
            for (int i = 0; i < PRE_KSW; ++i) {
                const int kstep = warp + 8 * i;
                const int k = (int)rank * Cs + kstep * 16;     // a 16-wide k step never straddles a 128-wide k block
                const uint32_t* src = reinterpret_cast<const uint32_t*>(xa + a16_index(t0 + 16 * sp + grp, k + tig * 2, TH));
                const bool ok = kstep < ksteps;
                af[i][0] = ok ? __ldcg(src) : 0u;                       // (t = grp,     k lo)
                af[i][1] = ok ? __ldcg(src + 32) : 0u;                  // (t = grp + 8, k lo)   +8 rows = 64 halves
                af[i][2] = ok ? __ldcg(src + TH * 4) : 0u;              // (t = grp,     k hi)   next k8 chunk = TH rows on
                af[i][3] = ok ? __ldcg(src + TH * 4 + 32) : 0u;         // (t = grp + 8, k hi)
            }
#pragma unroll
            for (int i = 0; i < PRE_KSW; ++i)
#pragma unroll
                for (int nt = 0; nt < PRE_NT2; ++nt) mma_16816(acc[nt], af[i], w1f[i][nt][0], w1f[i][nt][1]);
        }
#pragma unroll
        for (int nt = 0; nt < PRE_NT2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) red2[warp][(nt * 4 + e) * 32 + lane] = acc[nt][e];
        __syncthreads();
        for (int o = tid; o < PRE_NT2 * 4 * 32; o += PRE_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) s += red2[w][o];
            part[o] = s;
        }
        cl.sync();
        constexpr int PER = PRE_NT2 * 4 * 32 / PRE_CLUSTER;      // 48 outputs finalised per CTA
        if (tid < PER) {
            const int o = (int)rank * PER + tid;
            float v[PRE_CLUSTER];
#pragma unroll
            for (int r = 0; r < PRE_CLUSTER; ++r) v[r] = cl.map_shared_rank(part, r)[o];
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < PRE_CLUSTER; ++r) s += v[r];
            const int nt = o / 128, e = (o >> 5) & 3, ln = o & 31;
            const int t = t0 + (ln >> 2) + ((e & 2) ? 8 : 0);
            const int nrow = nt * 8 + (ln & 3) * 2 + (e & 1);
            const int n = g * RG + nrow;
            if (t < T && nrow < RG && n < NR) {
                const int j = n / Dm, nn = n - j * Dm;
                __half* dst = p.lora + (size_t)j * p.lora_stride;
                if (SPLIT) {
                    __half hi, lo;
                    split_h(apply_act(s, ACT_TANH), hi, lo);
                    dst[a16_index(t, nn, TH)] = hi;
                    dst[a16_index(t + 16, nn, TH)] = lo;
                } else {
                    dst[a16_index(t, nn, TH)] = f2h_sat(apply_act(s, ACT_TANH));
                }
            }
        }
    }
    trace_stamp(tr, 4);
    pre_grid_barrier(cl, rank, p.gbar + 32, nullptr, p.gbar, 2);      // also keeps every CTA alive until its peers finished reading `part`

    trace_stamp(tr, 5);
    // ---------------- phase 3: x_j = xx + sx * (mu_j + W2_j tanh_j) ----------------
    for (int q = 0; q < ngrp; ++q) {
        const int t0 = 16 * q;
        uint32_t af[PRE_TILES3][KD][4];
        float2 xx[PRE_TILES3][2], sx[PRE_TILES3][2];
        float acc3[SPLIT ? PRE_TILES3 : 1][4];
        if (SPLIT) {           // lo halves first (second 16-token tile of the LoRA matrices); the hi pass below adds to it
#pragma unroll
            for (int i = 0; i < PRE_TILES3; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc3[SPLIT ? i : 0][e] = 0.f;
#pragma unroll
            for (int i = 0; i < PRE_TILES3; ++i) {
                const bool ok = tj[i] >= 0;
                const uint32_t* src = reinterpret_cast<const uint32_t*>(p.lora + (size_t)(ok ? tj[i] : 0) * p.lora_stride +
                                                                        a16_index(t0 + 16 + grp, tig * 2, TH));
#pragma unroll
                for (int ks = 0; ks < KD; ++ks) {      // k16 step ks = k8 chunks 2 ks, 2 ks + 1 (TH rows x 8 halves each)
                    af[i][ks][0] = ok ? __ldcg(src + ks * TH * 8) : 0u;
                    af[i][ks][1] = ok ? __ldcg(src + ks * TH * 8 + 32) : 0u;
                    af[i][ks][2] = ok ? __ldcg(src + ks * TH * 8 + TH * 4) : 0u;
                    af[i][ks][3] = ok ? __ldcg(src + ks * TH * 8 + TH * 4 + 32) : 0u;
                }
            }
#pragma unroll
            for (int i = 0; i < PRE_TILES3; ++i)
#pragma unroll
                for (int ks = 0; ks < KD; ++ks) mma_16816(acc3[SPLIT ? i : 0], af[i][ks], w2f[i][ks][0], w2f[i][ks][1]);
        }
#pragma unroll
        for (int i = 0; i < PRE_TILES3; ++i) {
            const bool ok = tj[i] >= 0;
            const uint32_t* src = reinterpret_cast<const uint32_t*>(p.lora + (size_t)(ok ? tj[i] : 0) * p.lora_stride + a16_index(t0 + grp, tig * 2, TH));
#pragma unroll
            for (int ks = 0; ks < KD; ++ks) {
                af[i][ks][0] = ok ? __ldcg(src + ks * TH * 8) : 0u;                  // chunk 2*ks, t = grp
                af[i][ks][1] = ok ? __ldcg(src + ks * TH * 8 + 32) : 0u;             //             t = grp + 8
                af[i][ks][2] = ok ? __ldcg(src + ks * TH * 8 + TH * 4) : 0u;         // chunk 2*ks + 1
                af[i][ks][3] = ok ? __ldcg(src + ks * TH * 8 + TH * 4 + 32) : 0u;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int t = t0 + grp + 8 * h;
                const size_t at = (size_t)t * C + tc0[i] + tig * 2;
                const bool okt = ok && t < T;
                xx[i][h] = okt ? __ldcg(reinterpret_cast<const float2*>(p.ln.xx_out + at)) : make_float2(0.f, 0.f);
                sx[i][h] = okt ? __ldcg(reinterpret_cast<const float2*>(p.ln.sx_out + at)) : make_float2(0.f, 0.f);
            }
        }
#pragma unroll
        for (int i = 0; i < PRE_TILES3; ++i) {
            if (tj[i] < 0) continue;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            if (SPLIT) {
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[e] = acc3[SPLIT ? i : 0][e];
            }
#pragma unroll
            for (int ks = 0; ks < KD; ++ks) mma_16816(acc, af[i][ks], w2f[i][ks][0], w2f[i][ks][1]);
            __half* outp = p.out[tj[i]];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int t = t0 + grp + 8 * h;
                if (t >= T) continue;
                const float y0 = xx[i][h].x + sx[i][h].x * (mu3[i].x + acc[2 * h]);
                const float y1 = xx[i][h].y + sx[i][h].y * (mu3[i].y + acc[2 * h + 1]);
                if (SPLIT) {
                    uint32_t hi, lo;
                    split_pack_h2(y0, y1, hi, lo);
                    *reinterpret_cast<uint32_t*>(outp + a16_index(t, tc0[i] + tig * 2, TH)) = hi;
                    *reinterpret_cast<uint32_t*>(outp + a16_index(t + 16, tc0[i] + tig * 2, TH)) = lo;
                } else {
                    *reinterpret_cast<uint32_t*>(outp + a16_index(t, tc0[i] + tig * 2, TH)) = pack_h2(y0, y1);
                }
            }
        }
    }
    trace_stamp(tr, 7);
}

}  // namespace b200
