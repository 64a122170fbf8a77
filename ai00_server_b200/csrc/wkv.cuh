// WKV recurrences: v5 / v6 multi-head state update and v7 delta rule, fused with the per-head
// GroupNorm (eps 64e-5), the v7 bonus term and the output gate.
//
// Replaces web-rwkv's `time_mix_v5` / `time_mix_v6` / `time_mix_v7` + `group_norm` WGSL
// dispatches under `Runtime::infer` (reference run.rs:1143; SURVEY.md §2.2 K6/K6'/K7, math in
// App. A / App. B).
//
// One 128-thread CTA per (head, step entry).  The 64x64 f32 head state (16 KB) lives in HBM as
// M[value][key] for every version (v6's S[key][value] is stored transposed; the API layout is
// restored by the state import/export kernels), so that
//   * each thread owns a 4(value) x 8(key) patch: 8 coalesced 16-byte accesses, rows moved as full
//     256-byte runs;
//   * every reduction of the recurrence runs over the KEY index = across the 8 lanes that share a
//     value row -> pure shuffles, no shared-memory round trip:
//       v5/v6: out[v] = sum_k r[k] * (u[k] k[k] v[v] + M[v][k]);  M[v][k] = k[k] v[v] + w[k] M[v][k]
//       v7:    sa[v]  = sum_k M[v][k] * (-kk[k]);
//              M[v][k] = M[v][k] w[k] + sa[v] (kk[k] a[k]) + v[v] k[k];   out[v] = sum_k M[v][k] r[k]
//   * state is read once and written once per step, the recurrence loops over the slot's tokens
//     with the state in registers (prefill chunks).
// Output: f16( GroupNorm(out) [+ bonus] * gate ) (or its hi + lo split) written straight into the
// A16 operand of the output projection.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int WKV_N = 64;          // head size (all supported RWKV v5/v6/v7 models)
constexpr float GN_EPS = 64e-5f;

struct WkvParams {
    int version;            // 5, 6, 7
    int ld;                 // row stride of r/k/v/g/w/a/nu (floats) = local channels
    MetaView meta;
    float* state;           // [S][H][64][64] this layer, M[value][key]
    int H;                  // local heads
    const float* r;
    const float* k;
    const float* v;
    const float* g;         // v5/v6: silu(gate proj); v7: gate LoRA output
    const float* w;         // [T, ld] decay in (0,1) (v6/v7); null for v5
    const float* w_static;  // [ld] v5 decay exp(-exp(time_decay))
    const float* u;         // [ld] v5/v6 time_first
    const float* lnx_w;
    const float* lnx_b;
    // v7
    const float* a;         // [T, ld] in-context learning rate
    const float* nu;        // [T, ld] value-residual gate (layers > 0)
    float* v_first;         // [T, ld] layer 0 writes, later layers read
    int layer0;
    const float* k_k;
    const float* k_a;
    const float* r_k;
    __half* out;            // A16 [T, ld]
    int kq_tile;
    // v6 decay fold (null wd2t: off): decay LoRA stage 2 evaluated inside the WKV kernel
    const __half* wd2t;    // [H][Dd][64] f16: time_decay_w2 rows of each head, k-major
    const float* decay_bias;    // [ld] time_decay
    const __half* d1;       // A16 [T, Dd]: tanh(time_decay_w1 @ xw)
    int d1_kq;
    int Dd;
    unsigned long long* trace;  // profiling aid (null in production)
    // snapshot steps (wkv_kernel<..., SNAP>): [T] snapshot record of each token row or null (b200rwkv_infer_snapshots); the
    // state after that token goes to record + snap_off + head * 64 * 64, in the layout of `state`
    float* const* snap_rec;
    size_t snap_off;
};

struct WkvShared {
    float r[WKV_N], k[WKV_N], v[WKV_N], w[WKV_N], b[WKV_N], o[WKV_N];
    float red[4];
};

// Runs the recurrence for `nt` tokens starting at token index t0 on head h with the state patch
// m[4][KC] in registers.  `w_local`: optional shared-memory decay rows [token][64] (the v6 decay
// fold) indexed from local token `lt0`.
// `pre`: optional shared-memory copy of the head's per-token vectors, [array][token][64] with arrays
// r, k, v, g (, w, a, nu for v7) and `pre_stride` floats between arrays (staged runs: gathered in
// one batch of loads so the per-token loop never waits on L2).
// KC: key columns per thread (8: 128 threads per head); the thread's patch is m[e][f] = M[4*ig + e][KC*j4 + f].
template <int VER, int KC = 8, bool SPLIT = false, bool SNAP = false>
__device__ __forceinline__ void wkv_slot(const WkvParams& p, const int h, const int t0, const int nt, float (&m)[4][KC],
                                         WkvShared& sm, const float* w_local, const int lt0, const float* pre = nullptr,
                                         const int pre_stride = 0, const float* statics = nullptr) {
    // `statics`: optional shared-memory copy of this head's [ln_x weight 64][ln_x bias 64][time_first 64], staged by the
    // caller before it waited on the producer kernel (keeps three L2 round trips off the per-step chain)
    const int tid = (int)threadIdx.x;
    constexpr int LANES = WKV_N / KC;  // threads that share a value row (reduction width)
    const int ig = tid / LANES;        // value rows 4*ig .. 4*ig+3
    const int j4 = tid % LANES;        // key cols  KC*j4 .. KC*j4+KC-1
    const int ch = h * WKV_N;          // channel base of this head
    float u4[KC];
#pragma unroll
    for (int f = 0; f < KC; ++f) u4[f] = 0.f;
    if (VER != 7) {
#pragma unroll
        for (int f = 0; f < KC; ++f) u4[f] = statics ? statics[2 * WKV_N + j4 * KC + f] : p.u[ch + j4 * KC + f];
    }
    for (int tt = 0; tt < nt; ++tt) {
        const int t = t0 + tt;
        const size_t row = (size_t)t * p.ld + ch;
        // ---- per-token head vectors -> shared ----
        if (tid < WKV_N) {
            const int c = tid;
            const int pi = (lt0 + tt) * WKV_N + c;
            float r = pre ? pre[pi] : p.r[row + c];
            float k = pre ? pre[pre_stride + pi] : p.k[row + c];
            float v = pre ? pre[2 * pre_stride + pi] : p.v[row + c];
            float w;
            if (VER == 5) w = p.w_static[ch + c];
            else if (w_local) w = w_local[pi];
            else w = pre ? pre[4 * pre_stride + pi] : p.w[row + c];
            if (VER == 7) {
                const float a = pre ? pre[5 * pre_stride + pi] : p.a[row + c];
                float kk = k * p.k_k[ch + c];
                // l2 norm over the head: two warps
                float ss = warp_sum(kk * kk);
                if ((tid & 31) == 0) sm.red[tid >> 5] = ss;
                asm volatile("bar.sync 2, 64;" ::: "memory");
                ss = sm.red[0] + sm.red[1];
                kk = kk / fmaxf(sqrtf(ss), 1e-12f);
                k = k * (1.f + (a - 1.f) * p.k_a[ch + c]);
                if (p.layer0) p.v_first[row + c] = v;
                else v = v + (p.v_first[row + c] - v) * (pre ? pre[6 * pre_stride + pi] : p.nu[row + c]);
                float bonus = warp_sum(r * k * p.r_k[ch + c]);
                if ((tid & 31) == 0) sm.red[2 + (tid >> 5)] = bonus;
                sm.b[c] = kk * a;       // kk (.) a
                sm.o[c] = -kk;          // reuse o as -kk until the output phase
            }
            sm.r[c] = r; sm.k[c] = k; sm.v[c] = v; sm.w[c] = w;
        }
        __syncthreads();

        float rr[KC], kk_[KC], ww[KC];
#pragma unroll
        for (int f = 0; f < KC; ++f) { rr[f] = sm.r[j4 * KC + f]; kk_[f] = sm.k[j4 * KC + f]; ww[f] = sm.w[j4 * KC + f]; }
        float o[4];
        if (VER != 7) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float vv = sm.v[ig * 4 + e];
                float* me = m[e];
                float acc = 0.f;
#pragma unroll
                for (int f = 0; f < KC; ++f) {
                    const float kv = kk_[f] * vv;
                    acc += rr[f] * (u4[f] * kv + me[f]);
                    me[f] = kv + ww[f] * me[f];
                }
                o[e] = acc;
            }
        } else {
            float nk[KC], ka[KC];
#pragma unroll
            for (int f = 0; f < KC; ++f) { nk[f] = sm.o[j4 * KC + f]; ka[f] = sm.b[j4 * KC + f]; }
            float sa[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float* me = m[e];
                float s_ = 0.f;
#pragma unroll
                for (int f = 0; f < KC; f += 4) s_ += (me[f] * nk[f] + me[f + 1] * nk[f + 1]) + (me[f + 2] * nk[f + 2] + me[f + 3] * nk[f + 3]);
                sa[e] = s_;
            }
#pragma unroll
            for (int off = LANES / 2; off > 0; off >>= 1)
#pragma unroll
                for (int e = 0; e < 4; ++e) sa[e] += __shfl_xor_sync(0xffffffffu, sa[e], off);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float vv = sm.v[ig * 4 + e];
                float* me = m[e];
                float acc = 0.f;
#pragma unroll
                for (int f = 0; f < KC; ++f) {
                    me[f] = me[f] * ww[f] + sa[e] * ka[f] + vv * kk_[f];
                    acc += me[f] * rr[f];
                }
                o[e] = acc;
            }
        }
        if (SNAP) {         // the state after token t, for a snapshot of it; the registers go on unchanged
            float* rec = p.snap_rec[t];
            if (rec) {
                float* Ms = rec + p.snap_off + (size_t)h * (WKV_N * WKV_N);
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int q = 0; q < KC / 4; ++q)
                        __stcs(reinterpret_cast<float4*>(Ms + (ig * 4 + e) * WKV_N + j4 * KC + q * 4),
                               make_float4(m[e][q * 4], m[e][q * 4 + 1], m[e][q * 4 + 2], m[e][q * 4 + 3]));
            }
        }
#pragma unroll
        for (int off = LANES / 2; off > 0; off >>= 1)
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] += __shfl_xor_sync(0xffffffffu, o[e], off);
        __syncthreads();              // all reads of sm.o (-kk) done before it is overwritten
        if (j4 == 0) {
#pragma unroll
            for (int e = 0; e < 4; ++e) sm.o[ig * 4 + e] = o[e];
        }
        __syncthreads();

        // ---- GroupNorm over the head + gate, warp 0: 2 channels per lane ----
        if (tid < 32) {
            const float x0 = sm.o[tid], x1 = sm.o[tid + 32];
            const float mean = warp_sum(x0 + x1) * (1.f / WKV_N);
            const float d0 = x0 - mean, d1 = x1 - mean;
            const float var = warp_sum(d0 * d0 + d1 * d1) * (1.f / WKV_N);
            const float rstd = 1.0f / sqrtf(var + GN_EPS);
            const float lw0 = statics ? statics[tid] : p.lnx_w[ch + tid], lw1 = statics ? statics[tid + 32] : p.lnx_w[ch + tid + 32];
            const float lb0 = statics ? statics[WKV_N + tid] : p.lnx_b[ch + tid];
            const float lb1 = statics ? statics[WKV_N + tid + 32] : p.lnx_b[ch + tid + 32];
            float y0 = d0 * rstd * lw0 + lb0;
            float y1 = d1 * rstd * lw1 + lb1;
            if (VER == 7) {
                const float bonus = sm.red[2] + sm.red[3];
                y0 += bonus * sm.v[tid];
                y1 += bonus * sm.v[tid + 32];
            }
            const int gi = (lt0 + tt) * WKV_N + tid;
            y0 *= pre ? pre[3 * pre_stride + gi] : p.g[row + tid];
            y1 *= pre ? pre[3 * pre_stride + gi + 32] : p.g[row + tid + 32];
            if (SPLIT) {       // split operand of the output projection (common.cuh split_h): lo halves in the second token tile
                __half h0, l0, h1, l1;
                split_h(y0, h0, l0);
                split_h(y1, h1, l1);
                p.out[a16_index(t, ch + tid, p.kq_tile)] = h0;
                p.out[a16_index(t, ch + tid + 32, p.kq_tile)] = h1;
                p.out[a16_index(t + 16, ch + tid, p.kq_tile)] = l0;
                p.out[a16_index(t + 16, ch + tid + 32, p.kq_tile)] = l1;
            } else {
                p.out[a16_index(t, ch + tid, p.kq_tile)] = f2h_sat(y0);
                p.out[a16_index(t, ch + tid + 32, p.kq_tile)] = f2h_sat(y1);
            }
        }
        __syncthreads();              // shared vectors are rewritten by the next token
    }
}

// Stand-alone kernel, one CTA of 128 threads per (head, slot); each thread owns a 4 x 8 patch of the state.
// Shape: 64 heads x 16 slots = 1024 CTAs must be ONE wave (measured: with 256 threads x 64 registers only 592 fit and the
// second wave doubled the kernel), i.e. <= 72 registers at 7 CTAs per SM with half of them holding state.
// A decode step is a latency chain, not bandwidth (16 KB of state per CTA), so everything no kernel of this step writes --
// the decay-LoRA slice, ln_x, time_first, the step metadata, and the state patch itself -- is requested BEFORE
// griddepcontrol.wait, and after it one batch of loads brings the head's r/k/v/g(/w/a/nu) rows of up to WKV_STAGE_TOK
// tokens and the decay-LoRA inputs; longer slots (prefill chunks) read per token instead.
constexpr int WKV_SA_THREADS = 128;
constexpr int WKV_SA_KC = 8;
constexpr int WKV_STAGE_TOK = 4;
constexpr int WKV_STAGE_ARRAYS = 7;      // r, k, v, g, w, a, nu

__host__ __device__ inline int wkv_stage_arrays(int ver, bool fold) { return ver == 7 ? 7 : ((ver == 6 && !fold) ? 5 : 4); }

// dynamic shared memory: [fold only: [Dd][64] halves (k-major slice of time_decay_w2) | [WKV_STAGE_TOK][64] floats (decays) |
// [WKV_STAGE_TOK][Dd] halves | [2][64] floats] | staged rows [arrays][WKV_STAGE_TOK][64] floats | statics [3][64] floats
__host__ __device__ inline size_t wkv_smem_bytes(int ver, bool fold, int Dd, int max_tokens, bool split = false) {
    size_t b = 0;
    (void)max_tokens;      // decay rows are kept for the staged tokens only; longer runs fold one token at a time
    if (fold) b += (size_t)WKV_N * Dd * 2 + (size_t)WKV_STAGE_TOK * WKV_N * 4 + ((((size_t)WKV_STAGE_TOK * Dd * 2 * (split ? 2 : 1)) + 15) & ~(size_t)15) + 2 * WKV_N * 4;
    b += (size_t)wkv_stage_arrays(ver, fold) * WKV_STAGE_TOK * WKV_N * 4 + 3 * WKV_N * 4 + 64;
    return b;
}

// SPLIT (opt-in B200RWKV_SPLIT_ACT=1): the decay-LoRA input and the output are split operands (hi + lo f16 pairs).
// SNAP: a step that holds snapshots also stores the state after every token that carries one (WkvParams::snap_rec).
template <int VER, bool SPLIT = false, bool SNAP = false>
__global__ void __launch_bounds__(WKV_SA_THREADS, 7) wkv_kernel(const __grid_constant__ WkvParams p, const int max_tokens) {
    constexpr int KC = WKV_SA_KC, LANES = WKV_N / KC, NT = WKV_SA_THREADS;
    __shared__ WkvShared sm;
    extern __shared__ __align__(16) uint8_t wkv_dyn[];
    trace_stamp(p.trace, 0);
    pdl_launch_dependents();
    const int si = blockIdx.y;
    const int h = blockIdx.x;
    const int tid = threadIdx.x;
    const int ig = tid / LANES, j4 = tid % LANES;
    const int ch = h * WKV_N;
    const bool fold = (VER == 6) && p.wd2t != nullptr;
    const int Dd = fold ? p.Dd : 0;
    uint8_t* dyn = wkv_dyn;
    __half* wt = reinterpret_cast<__half*>(dyn);
    float* wl = nullptr;
    __half* ds = nullptr;
    float* part = nullptr;
    if (fold) {
        wl = reinterpret_cast<float*>(dyn + (size_t)WKV_N * Dd * 2);
        ds = reinterpret_cast<__half*>(wl + (size_t)WKV_STAGE_TOK * WKV_N);
        part = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ds) + ((((size_t)WKV_STAGE_TOK * Dd * 2 * (SPLIT ? 2 : 1)) + 15) & ~(size_t)15));
        dyn = reinterpret_cast<uint8_t*>(part + 2 * WKV_N);
    }
    const int na = wkv_stage_arrays(VER, fold);
    float* pre_s = reinterpret_cast<float*>(dyn);
    float* statics = pre_s + na * WKV_STAGE_TOK * WKV_N;
    // ---- before the wait: weights and step metadata ----
    if (fold) {
        const uint4* src = reinterpret_cast<const uint4*>(p.wd2t + (size_t)h * WKV_N * Dd);
        uint4* dst = reinterpret_cast<uint4*>(wt);
        for (int i = tid; i < WKV_N * Dd / 8; i += NT) dst[i] = src[i];
    }
    for (int i = tid; i < 3 * WKV_N; i += NT) {
        const int a = i >> 6, c = i & (WKV_N - 1);
        float v = 0.f;
        if (a == 0) v = p.lnx_w[ch + c];
        else if (a == 1) v = p.lnx_b[ch + c];
        else if (VER != 7) v = p.u[ch + c];
        statics[i] = v;
    }
    const float bias = fold ? p.decay_bias[ch + (tid & (WKV_N - 1))] : 0.f;
    const int nslots = p.meta.nslots();
    const bool live = si < nslots;
    const int slot = live ? p.meta.slot_id()[si] : 0;
    const int t0 = live ? p.meta.slot_start()[si] : 0;
    const int nt = live ? p.meta.slot_count()[si] : 0;
    // The state patch is requested BEFORE the wait as well: no kernel of this step but this one touches this layer's WKV
    // state, and CTAs that become resident while the slowest CTAs of the preceding projection are still finishing (its
    // tail skews by several microseconds) spend that time pulling their 16 KB from HBM instead of idling.
    float* M = p.state + ((size_t)slot * p.H + h) * (WKV_N * WKV_N);
    float m[4][KC];
    if (live) {
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int q = 0; q < KC / 4; ++q) {
                const float4 v4 = __ldcs(reinterpret_cast<const float4*>(M + (ig * 4 + e) * WKV_N + j4 * KC + q * 4));
                m[e][q * 4] = v4.x; m[e][q * 4 + 1] = v4.y; m[e][q * 4 + 2] = v4.z; m[e][q * 4 + 3] = v4.w;
            }
    }
    pdl_wait();
    trace_stamp(p.trace, 1);
    if (!live) return;

    // ---- one batch of loads: staged rows, decay-LoRA inputs ----
    const bool staged = nt <= WKV_STAGE_TOK;
    if (staged) {
        constexpr int UMAX = WKV_STAGE_ARRAYS * WKV_STAGE_TOK * WKV_N / NT;      // 14
        const int per = nt * WKV_N, total = na * per;
        const int ndd = fold ? nt * Dd : 0;
        // two half batches keep the register peak below the one-wave budget
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            float val[UMAX / 2];
#pragma unroll
            for (int u = 0; u < UMAX / 2; ++u) {
                const int i = tid + (half * (UMAX / 2) + u) * NT;
                val[u] = 0.f;
                if (i < total) {
                    const int a = i / per, rem = i - a * per;
                    const size_t at = (size_t)(t0 + (rem >> 6)) * p.ld + ch + (rem & (WKV_N - 1));
                    const float* src = a == 0 ? p.r : a == 1 ? p.k : a == 2 ? p.v : a == 3 ? p.g : a == 4 ? p.w : a == 5 ? p.a : p.nu;
                    if (src) val[u] = src[at];
                }
            }
#pragma unroll
            for (int u = 0; u < UMAX / 2; ++u) {
                const int i = tid + (half * (UMAX / 2) + u) * NT;
                if (i < total) {
                    const int a = i / per, rem = i - a * per;
                    pre_s[a * (WKV_STAGE_TOK * WKV_N) + rem] = val[u];
                }
            }
        }
        for (int i = tid; i < ndd; i += NT) {
            const int tt = i / Dd;
            ds[i] = p.d1[a16_index(t0 + tt, i - tt * Dd, p.d1_kq)];
        }
        if (SPLIT)
            for (int i = tid; i < ndd; i += NT) {
                const int tt = i / Dd;
                ds[WKV_STAGE_TOK * Dd + i] = p.d1[a16_index(t0 + tt + 16, i - tt * Dd, p.d1_kq)];
            }
    }

    // w[t][c] = exp(-exp(time_decay[c] + sum_k Wd2[c][k] * tanh(Wd1 xw)[t][k]))   (SURVEY.md App. A), for the token whose
    // decay-LoRA input sits at `dt` (hi) / `dt + WKV_STAGE_TOK * Dd` (lo halves of split operands), into wl[slot_tok][64]
    auto fold_token = [&](const __half* dt, const int slot_tok) {
        const int c = tid & (WKV_N - 1), qk = tid >> 6;
        const int kq0 = qk * (Dd >> 1), kq1 = kq0 + (Dd >> 1);
        float acc0 = 0.f, acc1 = 0.f;
        if (SPLIT) {
            const __half* dl = dt + WKV_STAGE_TOK * Dd;
            for (int k = kq0; k < kq1; k += 2) {
                acc0 = fmaf(__half2float(wt[k * WKV_N + c]), __half2float(dt[k]) + __half2float(dl[k]), acc0);
                acc1 = fmaf(__half2float(wt[(k + 1) * WKV_N + c]), __half2float(dt[k + 1]) + __half2float(dl[k + 1]), acc1);
            }
        } else {
            for (int k = kq0; k < kq1; k += 2) {
                acc0 = fmaf(__half2float(wt[k * WKV_N + c]), __half2float(dt[k]), acc0);
                acc1 = fmaf(__half2float(wt[(k + 1) * WKV_N + c]), __half2float(dt[k + 1]), acc1);
            }
        }
        part[qk * WKV_N + c] = acc0 + acc1;
        __syncthreads();
        if (tid < WKV_N) wl[slot_tok * WKV_N + c] = expf(-expf(bias + (part[c] + part[WKV_N + c])));
    };
    if (staged || !fold) {
        if (fold)
            for (int tt = 0; tt < nt; ++tt) {
                __syncthreads();
                fold_token(ds + tt * Dd, tt);
            }
        __syncthreads();
        wkv_slot<VER, KC, SPLIT, SNAP>(p, h, t0, nt, m, sm, fold ? wl : nullptr, 0, staged ? pre_s : nullptr, WKV_STAGE_TOK * WKV_N, statics);
    } else {
        // long run of one slot (prefill chunk): token by token, the decay row of one token at a time
        for (int tt = 0; tt < nt; ++tt) {
            __syncthreads();
            for (int k = tid; k < Dd; k += NT) ds[k] = p.d1[a16_index(t0 + tt, k, p.d1_kq)];
            if (SPLIT)
                for (int k = tid; k < Dd; k += NT) ds[WKV_STAGE_TOK * Dd + k] = p.d1[a16_index(t0 + tt + 16, k, p.d1_kq)];
            __syncthreads();
            fold_token(ds, 0);
            __syncthreads();
            wkv_slot<VER, KC, SPLIT, SNAP>(p, h, t0 + tt, 1, m, sm, wl, 0, nullptr, WKV_STAGE_TOK * WKV_N, statics);
        }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int q = 0; q < KC / 4; ++q)
            __stcs(reinterpret_cast<float4*>(M + (ig * 4 + e) * WKV_N + j4 * KC + q * 4),
                   make_float4(m[e][q * 4], m[e][q * 4 + 1], m[e][q * 4 + 2], m[e][q * 4 + 3]));
    trace_stamp(p.trace, 7);
}

}  // namespace b200
