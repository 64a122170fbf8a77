// Residual update + LayerNorm + token shift + static lerps, one 256-thread group per token.
//
// Replaces web-rwkv's `layer_norm`, `token_shift` and `add` WGSL dispatches on the path
// `Runtime::infer` (reference run.rs:1143; SURVEY.md §2.2 K1-K3, App. A/B).  Fused so the
// residual stream makes one HBM/L2 round trip per half-layer:
//     x_out = x_in + gate (.) sum_p part[p]            (projection results of the previous
//                                                       half-layer, one partial per TP rank)
//     xx    = LN(x_out)                                 eps 1e-5
//     prev  = first token of its slot ? shift_state[slot] : LN(x_out[t-1])   (recomputed)
//     sx    = prev - xx
//     mix_j = f16(xx + sx * mu_j)  -> A16 operand buffers of the following projections
// The shift state of the PREVIOUS LN stage is committed here (dst <- last token's xx), which
// keeps every state write strictly after all reads of the old value with no extra launch.
//
// Code shape: only a handful of CTAs run these rows and everything they touch sits at L2 latency
// (~0.5 us per dependent round trip), so the row lives in registers and every batch of loads is
// issued together; parameters that do not depend on the phase are requested before the reductions.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int LN_THREADS = 256;
constexpr int LN_MAXC = 8192;       // largest row the stand-alone kernels buffer
constexpr float LN_EPS = 1e-5f;

struct LnMixParams {
    const float* x_in;      // [T, C]
    float* x_out;           // [T, C] (may alias x_in only when n_parts == 0)
    int C;
    MetaView meta;
    int n_parts;
    const float* parts[8];  // [T, C] each
    int n_gate;             // 0 = no gate; else column-blocked gate, one block per TP rank
    int gate_cl;            // columns per gate block (C / n_gate)
    const float* gates[8];  // [T, gate_cl] each
    const float* ln_w;
    const float* ln_b;
    const float* shift_state;   // [S, C] rows of this layer / kind
    int n_mix;
    const float* mu[6];
    __half* mix_out[6];
    int kq_tile;            // th: token rows of this step's A16 operands (16 x token tiles; 32 with split operands)
    float* xx_out;          // [T, C]
    float* sx_out;          // [T, C] or null
    float* commit_dst;      // [S, C] or null
    const float* commit_src;    // [T, C]
    unsigned long long* trace;  // profiling aid (null in production)
    // LN1 of layer l + 1 only: slot l of the engine's per-layer hidden-row table (b200rwkv_keep_hidden_layers).  The slot
    // holds a [T, C] buffer that receives x_out (the residual stream after layer l) or null.  It changes only between
    // host-synchronous infer calls, so kernels read it before griddepcontrol.wait and the step graphs never change.
    float* const* hid_slot;
    // steps that hold snapshots (b200rwkv_infer_snapshots), else null: [T] snapshot record of each token row or null.  A
    // stage that commits a shift row also writes commit_src's row of every snapshot token to record + snap_off.
    float* const* snap_rec;
    size_t snap_off;
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void add4(float4& a, const float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

// residual source shared by the LN stages: x_in + gate (.) sum_p parts[p]
struct ResidualSrc {     // held by value: pointers into kernel-parameter space would turn into slow generic loads
    const float* x_in;
    int C, n_parts, n_gate, gate_cl;
    const float* parts[8];
    const float* gates[8];
};
template <typename P>
__device__ __forceinline__ ResidualSrc make_residual_src(const P& p) {
    ResidualSrc r;
    r.x_in = p.x_in; r.C = p.C; r.n_parts = p.n_parts; r.n_gate = p.n_gate; r.gate_cl = p.gate_cl;
#pragma unroll
    for (int i = 0; i < 8; ++i) { r.parts[i] = p.parts[i]; r.gates[i] = p.gates[i]; }
    return r;
}

// Row t of the updated residual into a[NV] (thread owns columns 4*(tid + 256 j)).  Memory-level
// parallelism is what matters here (a handful of CTAs, everything L2-latency bound): all loads of
// a batch (x + 4 partials, then 4 more partials + gate) are in flight together.
template <int NV>
__device__ __forceinline__ void residual_row(const ResidualSrc& r, const int t, float4 (&a)[NV]) {
    const int C = r.C;
    const size_t base = (size_t)t * C;
    float4 s[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        a[j] = (c < C) ? ld4(r.x_in + base + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        s[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (r.n_parts == 0) return;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        if (half * 4 >= r.n_parts) break;
        float4 v[4][NV];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                const int c = 4 * (threadIdx.x + LN_THREADS * j);
                v[q][j] = (half * 4 + q < r.n_parts && c < C) ? ld4(r.parts[half * 4 + q] + base + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
        for (int q = 0; q < 4; ++q)        // fixed order: deterministic, identical on all ranks
#pragma unroll
            for (int j = 0; j < NV; ++j) add4(s[j], v[q][j]);
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        if (r.n_gate > 0 && c < C) {
            const int gb = c / r.gate_cl;
            const float4 gt = ld4(r.gates[gb] + (size_t)t * r.gate_cl + (c - gb * r.gate_cl));
            s[j].x *= gt.x; s[j].y *= gt.y; s[j].z *= gt.z; s[j].w *= gt.w;
        }
        add4(a[j], s[j]);
    }
}

// two-pass mean / rstd of a row held in registers
template <int NV>
__device__ __forceinline__ void row_stats(const int C, const float4 (&a)[NV], float* red, float& mean, float& rstd) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) s += (a[j].x + a[j].y) + (a[j].z + a[j].w);
    mean = block_sum(s, red) / (float)C;
    float s2 = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        if (c < C) {
            const float dx = a[j].x - mean, dy = a[j].y - mean, dz = a[j].z - mean, dw = a[j].w - mean;
            s2 += (dx * dx + dy * dy) + (dz * dz + dw * dw);
        }
    }
    const float var = block_sum(s2, red) / (float)C;
    rstd = 1.0f / sqrtf(var + LN_EPS);
}

__device__ __forceinline__ float4 ln_apply(const float4 a, const float mean, const float rstd, const float4 w, const float4 b) {
    float4 o;
    o.x = (a.x - mean) * rstd * w.x + b.x;
    o.y = (a.y - mean) * rstd * w.y + b.y;
    o.z = (a.z - mean) * rstd * w.z + b.z;
    o.w = (a.w - mean) * rstd * w.w + b.w;
    return o;
}

// `hid`: null, or the [T, C] buffer that records this stage's updated residual (LnMixParams::hid_slot)
template <int NV>
__device__ __forceinline__ void ln_mix_row_nv(const LnMixParams& p, const int t, float* red, float* hid, unsigned long long* stamps = nullptr) {
    auto stamp = [&](int i) { if (stamps && threadIdx.x == 0) stamps[i] = globaltimer_ns(); };
    stamp(0);
    const int C = p.C;
    const int slot = p.meta.tok_slot()[t];
    const int prev_t = p.meta.tok_prev()[t];
    const bool last = p.meta.tok_last()[t] != 0;
    const ResidualSrc r = make_residual_src(p);
    float4 a[NV], w[NV], b[NV], pv[NV];
    stamp(1);
    residual_row<NV>(r, t, a);
    stamp(2);
    // LN parameters and the shift state do not depend on this phase: request them before the
    // reductions so their latency hides behind the two block sums
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        const bool ok = c < C;
        w[j] = ok ? ld4(p.ln_w + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        b[j] = ok ? ld4(p.ln_b + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        pv[j] = (ok && prev_t < 0) ? ld4(p.shift_state + (size_t)slot * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (p.x_out != p.x_in || p.n_parts > 0) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int c = 4 * (threadIdx.x + LN_THREADS * j);
            if (c < C) *reinterpret_cast<float4*>(p.x_out + (size_t)t * C + c) = a[j];
        }
    }
    if (hid) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int c = 4 * (threadIdx.x + LN_THREADS * j);
            if (c < C) *reinterpret_cast<float4*>(hid + (size_t)t * C + c) = a[j];
        }
    }
    float mean, rstd;
    stamp(3);
    row_stats<NV>(C, a, red, mean, rstd);
    stamp(4);
    if (prev_t >= 0) {          // multi-token slot (prefill): previous token's LN output, recomputed
        float pmean, prstd;
        residual_row<NV>(r, prev_t, pv);
        row_stats<NV>(C, pv, red, pmean, prstd);
#pragma unroll
        for (int j = 0; j < NV; ++j) pv[j] = ln_apply(pv[j], pmean, prstd, w[j], b[j]);
    }
    float4 sx[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        a[j] = ln_apply(a[j], mean, rstd, w[j], b[j]);       // xx
        sx[j].x = pv[j].x - a[j].x; sx[j].y = pv[j].y - a[j].y; sx[j].z = pv[j].z - a[j].z; sx[j].w = pv[j].w - a[j].w;
        if (c < C) {
            *reinterpret_cast<float4*>(p.xx_out + (size_t)t * C + c) = a[j];
            if (p.sx_out) *reinterpret_cast<float4*>(p.sx_out + (size_t)t * C + c) = sx[j];
            if (last && p.commit_dst)
                *reinterpret_cast<float4*>(p.commit_dst + (size_t)slot * C + c) = ld4(p.commit_src + (size_t)t * C + c);
        }
    }
    stamp(5);
#pragma unroll 1
    for (int m = 0; m < p.n_mix; ++m) {
        const float* mup = p.mu[m];
        __half* outp = p.mix_out[m];
        float4 mu[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int c = 4 * (threadIdx.x + LN_THREADS * j);
            mu[j] = (c < C) ? ld4(mup + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int c = 4 * (threadIdx.x + LN_THREADS * j);
            if (c < C) {
                uint2 o;
                o.x = pack_h2(a[j].x + sx[j].x * mu[j].x, a[j].y + sx[j].y * mu[j].y);
                o.y = pack_h2(a[j].z + sx[j].z * mu[j].z, a[j].w + sx[j].w * mu[j].w);
                *reinterpret_cast<uint2*>(outp + a16_index(t, c, p.kq_tile)) = o;
            }
        }
    }
}

// a snapshot step's copy of the shift row this stage commits: row t of `src` -> record + off (no-op for a null record)
__device__ __forceinline__ void snap_commit_row(float* rec, const size_t off, const float* src, const int t, const int C) {
    if (!rec) return;
    for (int c = 4 * (int)threadIdx.x; c < C; c += 4 * LN_THREADS)
        *reinterpret_cast<float4*>(rec + off + c) = ld4(src + (size_t)t * C + c);
}

__device__ __forceinline__ void ln_mix_row(const LnMixParams& p, const int t, float* red, float* hid, unsigned long long* stamps = nullptr) {
    const int nv = (p.C + 4 * LN_THREADS - 1) / (4 * LN_THREADS);
    if (nv <= 1) ln_mix_row_nv<1>(p, t, red, hid);
    else if (nv == 2) ln_mix_row_nv<2>(p, t, red, hid);
    else if (nv <= 4) ln_mix_row_nv<4>(p, t, red, hid, stamps);
    else ln_mix_row_nv<8>(p, t, red, hid);
    if (stamps && threadIdx.x == 0) stamps[6] = globaltimer_ns();
}

__global__ void __launch_bounds__(LN_THREADS) ln_mix_kernel(const __grid_constant__ LnMixParams p) {
    __shared__ float red[32];
    trace_stamp(p.trace, 0);
    pdl_launch_dependents();
    float* const hid = p.hid_slot ? *p.hid_slot : nullptr;
    pdl_wait();
    trace_stamp(p.trace, 1);
    const int t = blockIdx.x;
    if (t >= p.meta.T()) return;
    ln_mix_row(p, t, red, hid);
    if (p.snap_rec && p.commit_dst) snap_commit_row(p.snap_rec[t], p.snap_off, p.commit_src, t, p.C);
    trace_stamp(p.trace, 7);
}

// ---------------------------------------------------------------------------------------
// Embedding gather + LN0 (reference: web-rwkv embeds on the CPU and runs ln0 on the device,
// SURVEY.md §2.2 K1; here the f16 table lives in HBM and both are one kernel).
// ---------------------------------------------------------------------------------------
struct EmbedParams {
    const __half* emb;     // [V, C]
    int C, V;
    MetaView meta;
    const float* ln_w;
    const float* ln_b;
    float* x_out;          // [T, C]
};

template <int NV>
__device__ __forceinline__ void embed_row_nv(const EmbedParams& p, const int t, float* red) {
    const int C = p.C;
    int tok = p.meta.tok()[t];
    tok = min(max(tok, 0), p.V - 1);
    float4 a[NV], w[NV], b[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        if (c < C) {
            const uint2 raw = *reinterpret_cast<const uint2*>(p.emb + (size_t)tok * C + c);
            const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
            const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
            a[j] = make_float4(lo.x, lo.y, hi.x, hi.y);
            w[j] = ld4(p.ln_w + c);
            b[j] = ld4(p.ln_b + c);
        } else {
            a[j] = w[j] = b[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    float mean, rstd;
    row_stats<NV>(C, a, red, mean, rstd);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        if (c < C) *reinterpret_cast<float4*>(p.x_out + (size_t)t * C + c) = ln_apply(a[j], mean, rstd, w[j], b[j]);
    }
}

__device__ __forceinline__ void embed_row(const EmbedParams& p, const int t, float* red) {
    const int nv = (p.C + 4 * LN_THREADS - 1) / (4 * LN_THREADS);
    if (nv <= 1) embed_row_nv<1>(p, t, red);
    else if (nv == 2) embed_row_nv<2>(p, t, red);
    else if (nv <= 4) embed_row_nv<4>(p, t, red);
    else embed_row_nv<8>(p, t, red);
}

__global__ void __launch_bounds__(LN_THREADS) embed_ln0_kernel(const __grid_constant__ EmbedParams p) {
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const int t = blockIdx.x;
    if (t >= p.meta.T()) return;
    embed_row(p, t, red);
}

// ---------------------------------------------------------------------------------------
// Final residual update + ln_out for the rows that need logits (RnnOption::Last -> last token
// of the slot, Full -> every token; reference run.rs:812-822, 710-724), gathered into the A16
// operand of the head GEMM.  Also commits the last layer's channel-mix shift state.
// ---------------------------------------------------------------------------------------
struct LnOutParams {
    const float* x_in;      // [T, C]
    int C;
    MetaView meta;
    int n_parts;
    const float* parts[8];
    int n_gate;
    int gate_cl;
    const float* gates[8];
    const float* ln_w;
    const float* ln_b;
    __half* head_in;        // A16 [R rows, C]
    int kq_tile;
    float* commit_dst;
    const float* commit_src;
    float* hidden_out;      // optional [T, C]: updated residual (hidden states of the embeddings route)
    // steps that hold snapshots (b200rwkv_infer_snapshots), else null: the shift row of every snapshot token goes to its
    // record (LnMixParams::snap_rec), and the tokens snap_meta gives an output row also go, normalised, into row
    // snap_meta.tok_outrow()[t] of snap_head_in (snap_kq token rows): the operand of the snapshot rows' own head launch
    float* const* snap_rec;
    size_t snap_off;
    MetaView snap_meta;
    __half* snap_head_in;
    int snap_kq;
};

template <int NV, bool SPLIT = false>
__device__ __forceinline__ void ln_out_row_nv(const LnOutParams& p, const int t, float* red) {
    const int C = p.C;
    const int slot = p.meta.tok_slot()[t];
    const bool last = p.meta.tok_last()[t] != 0;
    const int row = p.meta.tok_outrow()[t];
    const int row2 = p.snap_head_in ? p.snap_meta.tok_outrow()[t] : -1;
    if (last && p.commit_dst) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int c = 4 * (threadIdx.x + LN_THREADS * j);
            if (c < C) *reinterpret_cast<float4*>(p.commit_dst + (size_t)slot * C + c) = ld4(p.commit_src + (size_t)t * C + c);
        }
    }
    if (row < 0 && row2 < 0 && !p.hidden_out) return;
    const ResidualSrc r = make_residual_src(p);
    float4 a[NV], w[NV], b[NV];
    residual_row<NV>(r, t, a);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        const bool ok = c < C;
        w[j] = ok ? ld4(p.ln_w + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        b[j] = ok ? ld4(p.ln_b + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok && p.hidden_out) *reinterpret_cast<float4*>(p.hidden_out + (size_t)t * C + c) = a[j];
    }
    if (row < 0 && row2 < 0) return;
    float mean, rstd;
    row_stats<NV>(C, a, red, mean, rstd);
    auto put = [&](__half* dst, const int rw, const int kq, const int c, const float4 y) {
        if (SPLIT) {       // rows of the head operand are output rows (<= 16 in a decode-shaped step); lo halves in tile 1
            uint2 hi, lo;
            split_pack_h2(y.x, y.y, hi.x, lo.x);
            split_pack_h2(y.z, y.w, hi.y, lo.y);
            *reinterpret_cast<uint2*>(dst + a16_index(rw, c, kq)) = hi;
            *reinterpret_cast<uint2*>(dst + a16_index(rw + 16, c, kq)) = lo;
        } else {
            uint2 o;
            o.x = pack_h2(y.x, y.y);
            o.y = pack_h2(y.z, y.w);
            *reinterpret_cast<uint2*>(dst + a16_index(rw, c, kq)) = o;
        }
    };
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int c = 4 * (threadIdx.x + LN_THREADS * j);
        if (c < C) {
            const float4 y = ln_apply(a[j], mean, rstd, w[j], b[j]);
            if (row >= 0) put(p.head_in, row, p.kq_tile, c, y);
            if (row2 >= 0) put(p.snap_head_in, row2, p.snap_kq, c, y);
        }
    }
}

template <bool SPLIT = false>
__device__ __forceinline__ void ln_out_row(const LnOutParams& p, const int t, float* red) {
    const int nv = (p.C + 4 * LN_THREADS - 1) / (4 * LN_THREADS);
    if (nv <= 1) ln_out_row_nv<1, SPLIT>(p, t, red);
    else if (nv == 2) ln_out_row_nv<2, SPLIT>(p, t, red);
    else if (nv <= 4) ln_out_row_nv<4, SPLIT>(p, t, red);
    else ln_out_row_nv<8, SPLIT>(p, t, red);
}

template <bool SPLIT = false>
__global__ void __launch_bounds__(LN_THREADS) ln_out_kernel(const __grid_constant__ LnOutParams p) {
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const int t = blockIdx.x;
    if (t >= p.meta.T()) return;
    ln_out_row<SPLIT>(p, t, red);
    if (p.snap_rec) snap_commit_row(p.snap_rec[t], p.snap_off, p.commit_src, t, p.C);
}

}  // namespace b200
