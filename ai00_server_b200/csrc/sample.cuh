// GPU front half of token sampling: penalties + allowed-token mask + bias + softmax + top-k, per slot, on the logits the
// head projection left in HBM.  Only <= 128 (token id, probability) pairs per slot cross PCIe.
//
// Replaces, for samplers that need only the head of the sorted distribution (Nucleus with top_k <= 128, greedy), what the
// reference does per generated token per slot (SURVEY.md §8f-1):
//   crates/ai00-core/src/run.rs:664-697   output.to_vec() (num_vocab f32 = 256 KiB D2H), Sampler::transform (penalties,
//                                         sampler/nucleus.rs:61-67), Formatter::transform (BNF mask, sampler/bnf.rs:37-40),
//                                         bias add (run.rs:679-681), softmax round trip (2 x 256 KiB, run.rs:1164-1190)
//   crates/ai00-core/src/sampler/nucleus.rs:69-80   full-vocabulary radix sort, `.rev().take(top_k)`
// The random draw, top_p cut, temperature and the penalty update (nucleus.rs:81-123) stay on the host: they need the
// sampler's state and RNG and touch <= top_k numbers.
//
// Order of the candidates: adjusted logit descending, token id ascending on ties -- a strict total order, so results are
// reproducible.  (The reference sorts probabilities with an unstable radix sort: any order of equal probabilities is a
// valid outcome there; this is one of them, because the probability is a non-decreasing function of the logit.)
//
// Shape: the vocabulary row (65536 f32 = 256 KB, L2 resident) is cut into 2048-element segments.
//   kernel 1 (grid = segments x rows): load, apply the two sparse lists and the mask, segment max / sum-exp, bitonic sort in
//            shared memory, keep the segment's best 128;
//   kernel 2 (grid = rows): combine the segment statistics into the softmax denominator (fixed order), merge the 32 sorted
//            lists pairwise -- the 128 best of two descending lists are first(a[i], b[127-i]), a bitonic sequence that seven
//            compare-exchange stages sort -- five rounds, then probabilities of the survivors.
// Nothing here is bandwidth: 16 rows x 256 KB from L2; two short launches.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int TOPK_MAX = 128;
constexpr int TOPK_SEG = 2048;            // elements per segment
constexpr int TOPK_SEG_THREADS = 256;
constexpr int TOPK_MAX_SEGS = 32;         // => num_vocab <= 65536
constexpr int TOPK_MERGE_THREADS = 1024;

// The rows to sample and their adjustments (run.rs:671-682), staged in one blob by the host; shared by both entry points.
struct SampleAdjust {
    const int* slot;            // [nrows]
    const int* pen_off;         // [nrows + 1]
    const unsigned* pen_tok;    // logits[tok] -= val   (entries of one row have distinct tokens)
    const float* pen_val;
    const int* bias_off;        // [nrows + 1]
    const unsigned* bias_tok;   // logits[tok] += val   (distinct tokens within a row)
    const float* bias_val;
    const unsigned* allow;      // optional [nrows][ceil(V / 32)]: bit = 1 -> token allowed; disallowed -> -inf
};

struct TopkParams {
    const float* keep;          // [S][V] last logits row of every slot
    int V, nseg;
    SampleAdjust adj;
    float* cand_x;              // [nrows][nseg][128]
    unsigned* cand_id;          // [nrows][nseg][128]
    float2* stats;              // [nrows][nseg] (max, sum exp(x - max))
    int top_k;
    unsigned* out_id;           // [nrows][top_k]
    float* out_p;               // [nrows][top_k]
};

// strict total order: larger logit first, then smaller id
__device__ __forceinline__ bool cand_before(const float xa, const unsigned ia, const float xb, const unsigned ib) {
    return xa > xb || (xa == xb && ia < ib);
}

// Adjusts segment `seg0 .. seg0 + TOPK_SEG` of row `row`, already loaded into sx (-inf past V), in place: penalties, the
// allowed-token mask, then bias -- the order of run.rs:671-682.  All TOPK_SEG_THREADS threads call it; it synchronises
// before it reads sx and before it returns.
__device__ __forceinline__ void adjust_segment(float* sx, const int seg0, const int V, const int row, const SampleAdjust& a) {
    const int tid = threadIdx.x;
    const unsigned* allow = a.allow ? a.allow + (size_t)row * ((V + 31) / 32) : nullptr;
    __syncthreads();
    // Sampler::transform: penalties (distinct tokens: race free)
    for (int e = a.pen_off[row] + tid; e < a.pen_off[row + 1]; e += TOPK_SEG_THREADS) {
        const unsigned t = a.pen_tok[e];
        if (t >= (unsigned)seg0 && t < (unsigned)(seg0 + TOPK_SEG) && t < (unsigned)V) sx[t - seg0] -= a.pen_val[e];
    }
    __syncthreads();
    // Formatter::transform: tokens the grammar does not allow
    if (allow) {
#pragma unroll
        for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) {
            const int li = tid + TOPK_SEG_THREADS * j, i = seg0 + li;
            if (i < V && !((allow[i >> 5] >> (i & 31)) & 1u)) sx[li] = -INFINITY;
        }
        __syncthreads();
    }
    // bias
    for (int e = a.bias_off[row] + tid; e < a.bias_off[row + 1]; e += TOPK_SEG_THREADS) {
        const unsigned t = a.bias_tok[e];
        if (t >= (unsigned)seg0 && t < (unsigned)(seg0 + TOPK_SEG) && t < (unsigned)V) sx[t - seg0] += a.bias_val[e];
    }
    __syncthreads();
}

// Softmax statistics of one adjusted segment in shared memory: (max, sum expf(x - max)), (-inf, 0) if every element is -inf.
// Element i always goes to thread i % TOPK_SEG_THREADS and the block reductions have a fixed shape, so the result depends
// only on the segment's values.
__device__ __forceinline__ float2 segment_stats(const float* sx, float* red) {
    const int tid = threadIdx.x;
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) mx = fmaxf(mx, sx[tid + TOPK_SEG_THREADS * j]);
    mx = block_max_any(mx, red);
    float s = 0.f;
    if (mx > -INFINITY) {
#pragma unroll
        for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) s += expf(sx[tid + TOPK_SEG_THREADS * j] - mx);
    }
    s = block_sum_any(s, red);
    return make_float2(mx, s);
}

// Bitonic sort of one segment in shared memory, best first (cand_before).  All TOPK_SEG_THREADS threads call it; it
// synchronises before it reads, not after its last stage.
__device__ __forceinline__ void sort_segment(float* sx, unsigned* sid) {
    const int tid = threadIdx.x;
    for (int k = 2; k <= TOPK_SEG; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
#pragma unroll
            for (int q = 0; q < TOPK_SEG / 2 / TOPK_SEG_THREADS; ++q) {
                const int t = tid + TOPK_SEG_THREADS * q;            // compare-exchange index 0 .. 1023
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)); // lower element of the pair
                const int l = i | j;
                const bool up = (i & k) == 0;                         // this block sorts best-first
                const float xa = sx[i], xb = sx[l];
                const unsigned ia = sid[i], ib = sid[l];
                const bool a_first = cand_before(xa, ia, xb, ib);
                if (a_first != up) { sx[i] = xb; sx[l] = xa; sid[i] = ib; sid[l] = ia; }
            }
        }
    }
}

// Merges the TOPK_MAX_SEGS sorted lists of TOPK_MAX candidates in shared memory into the best TOPK_MAX, in sx[0 .. 127] /
// sid[0 .. 127], in five rounds: lists a = 2 p s, b = (2 p + 1) s -> a.  All TOPK_MERGE_THREADS threads call it; it
// synchronises before it reads, not after its last stage.
__device__ __forceinline__ void merge_lists(float* sx, unsigned* sid) {
    const int tid = threadIdx.x;
    for (int s = 1; s < TOPK_MAX_SEGS; s <<= 1) {
        const int npair = TOPK_MAX_SEGS / (2 * s);
        __syncthreads();
        for (int t = tid; t < npair * TOPK_MAX; t += TOPK_MERGE_THREADS) {
            const int pr = t / TOPK_MAX, i = t % TOPK_MAX;
            const int a = (2 * pr) * s * TOPK_MAX + i, b = (2 * pr + 1) * s * TOPK_MAX + (TOPK_MAX - 1 - i);
            if (!cand_before(sx[a], sid[a], sx[b], sid[b])) { sx[a] = sx[b]; sid[a] = sid[b]; }
        }
        for (int j = TOPK_MAX / 2; j > 0; j >>= 1) {
            __syncthreads();
            for (int t = tid; t < npair * (TOPK_MAX / 2); t += TOPK_MERGE_THREADS) {
                const int pr = t / (TOPK_MAX / 2), u = t % (TOPK_MAX / 2);
                const int i = (2 * pr) * s * TOPK_MAX + (((u & ~(j - 1)) << 1) | (u & (j - 1)));
                const int l = i + j;
                const float xa = sx[i], xb = sx[l];
                const unsigned ia = sid[i], ib = sid[l];
                if (!cand_before(xa, ia, xb, ib)) { sx[i] = xb; sx[l] = xa; sid[i] = ib; sid[l] = ia; }
            }
        }
    }
}

__global__ void __launch_bounds__(TOPK_SEG_THREADS) topk_segment_kernel(const __grid_constant__ TopkParams p) {
    __shared__ float sx[TOPK_SEG];
    __shared__ unsigned sid[TOPK_SEG];
    __shared__ float red[32];
    const int seg = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    const int seg0 = seg * TOPK_SEG;
    const float* src = p.keep + (size_t)p.adj.slot[row] * p.V;
#pragma unroll
    for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) {
        const int li = tid + TOPK_SEG_THREADS * j, i = seg0 + li;
        sx[li] = (i < p.V) ? src[i] : -INFINITY;
        sid[li] = (i < p.V) ? (unsigned)i : 0xFFFFFFFFu;
    }
    adjust_segment(sx, seg0, p.V, row, p.adj);
    // segment statistics of the softmax
    const float2 st = segment_stats(sx, red);
    if (tid == 0) p.stats[(size_t)row * p.nseg + seg] = st;
    sort_segment(sx, sid);
    __syncthreads();
    if (tid < TOPK_MAX) {
        const size_t o = ((size_t)row * p.nseg + seg) * TOPK_MAX + tid;
        p.cand_x[o] = sx[tid];
        p.cand_id[o] = sid[tid];
    }
}

__global__ void __launch_bounds__(TOPK_MERGE_THREADS) topk_merge_kernel(const __grid_constant__ TopkParams p) {
    __shared__ float sx[TOPK_MAX_SEGS * TOPK_MAX];
    __shared__ unsigned sid[TOPK_MAX_SEGS * TOPK_MAX];
    __shared__ float s_m, s_inv;
    const int row = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < TOPK_MAX_SEGS * TOPK_MAX; i += TOPK_MERGE_THREADS) {
        const int sg = i / TOPK_MAX;
        const bool ok = sg < p.nseg;
        const size_t o = ((size_t)row * p.nseg + sg) * TOPK_MAX + (i % TOPK_MAX);
        sx[i] = ok ? p.cand_x[o] : -INFINITY;
        sid[i] = ok ? p.cand_id[o] : 0xFFFFFFFFu;
    }
    if (tid < 32) {
        // softmax denominator from the segment statistics, fixed order (lane = segment, xor tree)
        const float2 st = (tid < p.nseg) ? p.stats[(size_t)row * p.nseg + tid] : make_float2(-INFINITY, 0.f);
        const float M = warp_max(st.x);
        float sc = (st.x > -INFINITY) ? st.y * expf(st.x - M) : 0.f;
        sc = warp_sum(sc);
        if (tid == 0) { s_m = M; s_inv = 1.0f / sc; }
    }
    merge_lists(sx, sid);
    __syncthreads();
    if (tid < p.top_k) {
        // same expression as softmax_kernel (misc.cuh): exp(x - max) * (1 / sum)
        p.out_id[(size_t)row * p.top_k + tid] = sid[tid];
        p.out_p[(size_t)row * p.top_k + tid] = (sx[tid] > -INFINITY) ? expf(sx[tid] - s_m) * s_inv : 0.f;
    }
}

// ---------------------------------------------------------------------------------------
// Whole adjusted distribution (b200rwkv_sample_probs): for samplers that read every probability (Mirostat, Typical, Nucleus
// with top_k > 128), the vector run.rs:673-691 hands to Sampler::sample, softmax(logits - penalties, masked, + bias), written
// from the slot's kept row.  Any num_vocab; same segments, adjustment and segment statistics as topk_segment_kernel.
//   pass 1 (grid = segments x rows): load, adjust_segment, segment_stats; the adjusted segment goes to `out`;
//   pass 2 (grid = segments x rows): every CTA combines its row's segment statistics in a fixed order (lane g of warp 0
//            takes segments g, g + 32, ... in turn, then an xor tree), then writes expf(x - M) * (1 / S) over its segment
//            with float4 (rows of `out` are 16-byte aligned: ld = V rounded up to 4) and a scalar tail for V % 4.
// For num_vocab <= 65536 (at most 32 segments, one per lane) the combine and the expression are topk_merge_kernel's, so a
// candidate's probability from sample_topk equals this row's entry bit for bit.  A disallowed token is exactly 0; a row
// with every token disallowed is all zeros (sample_topk's probabilities on such a row are 0 as well).
// ---------------------------------------------------------------------------------------
struct ProbsParams {
    const float* keep;          // [S][V] last logits row of every slot
    int V, nseg, ld;            // ld: row stride of `out` in floats, V rounded up to a multiple of 4
    SampleAdjust adj;
    float* out;                 // [nrows][ld]: adjusted logits after pass 1, probabilities after pass 2
    float2* stats;              // [nrows][nseg] (max, sum exp(x - max))
};

__global__ void __launch_bounds__(TOPK_SEG_THREADS) probs_stats_kernel(const __grid_constant__ ProbsParams p) {
    __shared__ float sx[TOPK_SEG];
    __shared__ float red[32];
    const int seg = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    const int seg0 = seg * TOPK_SEG;
    const float* src = p.keep + (size_t)p.adj.slot[row] * p.V;
#pragma unroll
    for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) {
        const int li = tid + TOPK_SEG_THREADS * j, i = seg0 + li;
        sx[li] = (i < p.V) ? src[i] : -INFINITY;
    }
    adjust_segment(sx, seg0, p.V, row, p.adj);
    const float2 st = segment_stats(sx, red);
    if (tid == 0) p.stats[(size_t)row * p.nseg + seg] = st;
    float* dst = p.out + (size_t)row * p.ld;
#pragma unroll
    for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) {
        const int li = tid + TOPK_SEG_THREADS * j, i = seg0 + li;
        if (i < p.V) dst[i] = sx[li];
    }
}

__global__ void __launch_bounds__(TOPK_SEG_THREADS) probs_write_kernel(const __grid_constant__ ProbsParams p) {
    __shared__ float s_m, s_inv;
    const int seg = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    if (tid < 32) {
        const float2* st = p.stats + (size_t)row * p.nseg;
        float m = -INFINITY;
        for (int g = tid; g < p.nseg; g += 32) m = fmaxf(m, st[g].x);
        const float M = warp_max(m);
        float sc = 0.f;
        for (int g = tid; g < p.nseg; g += 32) {
            const float2 v = st[g];
            sc += (v.x > -INFINITY) ? v.y * expf(v.x - M) : 0.f;
        }
        sc = warp_sum(sc);
        if (tid == 0) { s_m = M; s_inv = 1.0f / sc; }
    }
    __syncthreads();
    const float M = s_m, inv = s_inv;
    float* x = p.out + (size_t)row * p.ld;
    float4* x4 = reinterpret_cast<float4*>(x);
    const int n4 = p.V >> 2;
    const int q1 = min(n4, (seg + 1) * (TOPK_SEG / 4));
    for (int q = seg * (TOPK_SEG / 4) + tid; q < q1; q += TOPK_SEG_THREADS) {
        float4 v = x4[q];
        v.x = (v.x > -INFINITY) ? expf(v.x - M) * inv : 0.f;
        v.y = (v.y > -INFINITY) ? expf(v.y - M) * inv : 0.f;
        v.z = (v.z > -INFINITY) ? expf(v.z - M) * inv : 0.f;
        v.w = (v.w > -INFINITY) ? expf(v.w - M) * inv : 0.f;
        x4[q] = v;
    }
    if (seg == p.nseg - 1 && tid < (p.V & 3)) {           // scalar tail
        const float v = x[4 * n4 + tid];
        x[4 * n4 + tid] = (v > -INFINITY) ? expf(v - M) * inv : 0.f;
    }
}

// ---------------------------------------------------------------------------------------
// Last logits row of every slot that produced one in this step -> keep[slot][V].  The rows of a step are overwritten by
// the next step, which may belong to other slots (the reference samples every slot in its own task while the infer loop
// goes on, run.rs:1230-1240), so the front half above reads from this per-slot copy.  Tensor parallel: rank 0 gathers the
// vocabulary shards of all ranks (rows complete after the step's last rendezvous).
// ---------------------------------------------------------------------------------------
struct KeepParams {
    const float* shard[8];      // [R][Vl] logits shard of every rank (peer mapped)
    int world, Vl, V;
    MetaView meta;
    float* keep;                // [S][V]
};
constexpr int KEEP_THREADS = 256;
constexpr int KEEP_CHUNKS = 8;

__global__ void __launch_bounds__(KEEP_THREADS) keep_rows_kernel(const __grid_constant__ KeepParams p) {
    pdl_launch_dependents();
    const int r = blockIdx.x;
    const int R = p.meta.R();
    const int t = (r < R) ? p.meta.out_tok()[r] : 0;
    const bool live = r < R && p.meta.tok_last()[t] != 0;
    const int slot = live ? p.meta.tok_slot()[t] : 0;
    pdl_wait();
    if (!live) return;
    float* dst = p.keep + (size_t)slot * p.V;
    const int n4 = p.Vl >> 2;
    const int i0 = blockIdx.y * KEEP_THREADS + threadIdx.x;
    for (int q = 0; q < p.world; ++q) {
        const float* s = p.shard[q] + (size_t)r * p.Vl;
        float* d = dst + (size_t)q * p.Vl;
        // Vl % 4 == 0: every row is 16-byte aligned on both sides.  Otherwise rows start anywhere: float4 loads, scalar stores
        // where the destination row is not aligned the same way, scalar loads where the source row is not aligned at all.
        const bool s_al = (reinterpret_cast<uintptr_t>(s) & 15) == 0, d_al = (reinterpret_cast<uintptr_t>(d) & 15) == 0;
        for (int i = i0; i < n4; i += KEEP_CHUNKS * KEEP_THREADS) {
            const float4 v = s_al ? __ldcg(reinterpret_cast<const float4*>(s) + i)
                                  : make_float4(__ldcg(s + 4 * i), __ldcg(s + 4 * i + 1), __ldcg(s + 4 * i + 2), __ldcg(s + 4 * i + 3));
            if (d_al) reinterpret_cast<float4*>(d)[i] = v;
            else { d[4 * i] = v.x; d[4 * i + 1] = v.y; d[4 * i + 2] = v.z; d[4 * i + 3] = v.w; }
        }
        if (i0 < (p.Vl & 3)) d[4 * n4 + i0] = __ldcg(s + 4 * n4 + i0);      // scalar tail
    }
}

// The logits row of every snapshot token of a step -> its snapshot (b200rwkv_infer_snapshots): src[t] is the step's output
// row of token t, or its row of the snapshot head launch; dst[t] the snapshot's row, or null.  One engine, all V columns.
struct SnapRowParams {
    const float* const* src;    // [rows of the step]
    float* const* dst;
    int V;
};

__global__ void __launch_bounds__(KEEP_THREADS) snap_rows_kernel(const __grid_constant__ SnapRowParams p) {
    pdl_launch_dependents();
    const int t = blockIdx.x;
    const float* s = p.src[t];
    float* d = p.dst[t];
    pdl_wait();
    if (!d) return;
    const int n4 = p.V >> 2;
    const int i0 = blockIdx.y * KEEP_THREADS + threadIdx.x;
    const bool al = ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0;
    for (int i = i0; i < n4; i += KEEP_CHUNKS * KEEP_THREADS) {
        const float4 v = al ? __ldcg(reinterpret_cast<const float4*>(s) + i)
                            : make_float4(__ldcg(s + 4 * i), __ldcg(s + 4 * i + 1), __ldcg(s + 4 * i + 2), __ldcg(s + 4 * i + 3));
        if (al) reinterpret_cast<float4*>(d)[i] = v;
        else { d[4 * i] = v.x; d[4 * i + 1] = v.y; d[4 * i + 2] = v.z; d[4 * i + 3] = v.w; }
    }
    if (i0 < (p.V & 3)) d[4 * n4 + i0] = __ldcg(s + 4 * n4 + i0);      // scalar tail
}

// ---------------------------------------------------------------------------------------
// Scoring (b200rwkv_infer_ex, B200RWKV_OPTION_SCORE): for each listed row, log softmax(row)[target] and the row's argmax
// (lowest id on ties, the sample_topk order), so a caller that wants the probability of a known continuation -- the
// reference's perplexity() and choose paths, run.rs:699-755 / 936-983 -- receives 8 bytes per token instead of a num_vocab
// f32 row.  One CTA per row; the row was just written by the head (L2 resident) or is a slot's kept row, and is read once.
//   score = (x_t - m) - logf(sum expf(x - m)),  m = row max   (the reference's exp(x) / sum exp(x), run.rs:738, overflows in
//   f32 above a logit of about 88; elsewhere the two agree to f32 rounding)
// Element i of the row always goes to thread (i / 4) % SCORE_THREADS, in the same order, whatever the row's address: the
// result of a row does not depend on where it sits in d_logits or which rows share the launch.  src == nullptr (a slot with
// no kept row): NaN and UINT32_MAX.  A NaN anywhere in the row makes the score NaN, as it makes softmax_kernel's row and the
// reference's exp(x) / sum exp(x) NaN; the argmax skips NaN entries (UINT32_MAX for a row of only NaN).  The NaN flag rides
// beside the sums and changes none of their arithmetic.
// ---------------------------------------------------------------------------------------
struct ScoreRow {
    const float* src;           // [V]
    unsigned target;            // token whose log-probability is wanted
    unsigned dst;               // index into score / argmax
};
struct ScoreParams {
    const ScoreRow* rows;
    int V;
    float* score;
    unsigned* argmax;
};
constexpr int SCORE_THREADS = 256;

struct ScoreAcc {
    float m, s;                 // running max, sum expf(x - m)
    float bx;                   // best logit, its lowest id
    unsigned bi;
    int nan;                    // a NaN was seen (every comparison below is false for one, so the sums skip it)
    __device__ __forceinline__ void add(const float x, const unsigned i) {
        nan |= x != x;
        if (x > m) { s = s * expf(m - x) + 1.f; m = x; }
        else if (x > -INFINITY) s += expf(x - m);
        if (x > bx || (x == bx && i < bi)) { bx = x; bi = i; }
    }
    __device__ __forceinline__ void merge(const ScoreAcc& o) {
        const float M = fmaxf(m, o.m);
        if (M > -INFINITY) s = (m > -INFINITY ? s * expf(m - M) : 0.f) + (o.m > -INFINITY ? o.s * expf(o.m - M) : 0.f);
        m = M;
        if (o.bx > bx || (o.bx == bx && o.bi < bi)) { bx = o.bx; bi = o.bi; }
        nan |= o.nan;
    }
    __device__ __forceinline__ ScoreAcc shfl_xor(const int lane_mask) const {
        return {__shfl_xor_sync(0xffffffffu, m, lane_mask), __shfl_xor_sync(0xffffffffu, s, lane_mask),
                __shfl_xor_sync(0xffffffffu, bx, lane_mask), __shfl_xor_sync(0xffffffffu, bi, lane_mask),
                __shfl_xor_sync(0xffffffffu, nan, lane_mask)};
    }
};

// score_rows_kernel's pass over a row, in two halves, for score_top_merge_kernel: the same element-to-thread map, additions
// and combine order, so both kernels find the same (m, s) bit for bit (tests/test_gpu_score_top.py holds them to it).
// score_row_warp: thread tid < SCORE_THREADS's share of the row, combined over its warp by an xor tree.  score_row_combine:
// warp 0 combines the SCORE_THREADS / 32 warps' results in the same way.  (score_rows_kernel keeps its own copy of these
// lines: calling these helpers from it changes its register allocation.)
__device__ __forceinline__ void score_row_warp(ScoreAcc& a, const float* s, const int V, const int tid) {
    const int n4 = V >> 2;
    if ((reinterpret_cast<uintptr_t>(s) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(s);
        for (int g = tid; g < n4; g += SCORE_THREADS) {
            const float4 v = __ldcg(s4 + g);
            a.add(v.x, 4 * g); a.add(v.y, 4 * g + 1); a.add(v.z, 4 * g + 2); a.add(v.w, 4 * g + 3);
        }
    } else {
        for (int g = tid; g < n4; g += SCORE_THREADS)
            for (int k = 0; k < 4; ++k) a.add(__ldcg(s + 4 * g + k), 4 * g + k);
    }
    if (tid < (V & 3)) a.add(__ldcg(s + 4 * n4 + tid), 4 * n4 + tid);      // scalar tail
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a.merge(a.shfl_xor(o));
}

__device__ __forceinline__ void score_row_combine(ScoreAcc& a, const ScoreAcc* red, const int tid) {
    a = (tid < SCORE_THREADS / 32) ? red[tid] : ScoreAcc{-INFINITY, 0.f, -INFINITY, 0xFFFFFFFFu, 0};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a.merge(a.shfl_xor(o));
}

__global__ void __launch_bounds__(SCORE_THREADS) score_rows_kernel(const __grid_constant__ ScoreParams p) {
    __shared__ ScoreAcc red[SCORE_THREADS / 32];
    const ScoreRow rw = p.rows[blockIdx.x];
    const int tid = threadIdx.x;
    if (rw.src == nullptr) {
        if (tid == 0) { p.score[rw.dst] = __int_as_float(0x7fc00000); p.argmax[rw.dst] = 0xFFFFFFFFu; }
        return;
    }
    ScoreAcc a{-INFINITY, 0.f, -INFINITY, 0xFFFFFFFFu, 0};
    const int n4 = p.V >> 2;
    const float* s = rw.src;
    if ((reinterpret_cast<uintptr_t>(s) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(s);
        for (int g = tid; g < n4; g += SCORE_THREADS) {
            const float4 v = __ldcg(s4 + g);
            a.add(v.x, 4 * g); a.add(v.y, 4 * g + 1); a.add(v.z, 4 * g + 2); a.add(v.w, 4 * g + 3);
        }
    } else {
        for (int g = tid; g < n4; g += SCORE_THREADS)
            for (int k = 0; k < 4; ++k) a.add(__ldcg(s + 4 * g + k), 4 * g + k);
    }
    if (tid < (p.V & 3)) a.add(__ldcg(s + 4 * n4 + tid), 4 * n4 + tid);      // scalar tail
    // fixed-order combine: xor tree inside each warp, then warp 0 over the warps' results
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a.merge(a.shfl_xor(o));
    if ((tid & 31) == 0) red[tid >> 5] = a;
    __syncthreads();
    if (tid < 32) {
        a = (tid < SCORE_THREADS / 32) ? red[tid] : ScoreAcc{-INFINITY, 0.f, -INFINITY, 0xFFFFFFFFu, 0};
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a.merge(a.shfl_xor(o));
        if (tid == 0) {
            p.score[rw.dst] = a.nan ? __int_as_float(0x7fc00000) : (__ldcg(s + rw.target) - a.m) - logf(a.s);
            p.argmax[rw.dst] = a.bi;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Top-n of every scored row (b200rwkv_score_top): the n best entries of each row score_rows_kernel scores, logit descending
// then id ascending (sample_topk's order on an unadjusted row), with logprob = (x - m) - logf(s) from the same (m, s) as the
// row's score, so the target's entry, when listed, equals its score bit for bit.  The row list, and so the launch shape, is
// the score launch's.
//   kernel 1 (grid = segments x rows): load a segment, NaN entries out of the ranking (sorted last, as padding is), bitonic
//            sort, keep the segment's best 128 -- topk_segment_kernel without adjustment or statistics;
//   kernel 2 (grid = rows): warps 0 .. 7 run the score pass over the row while the others load the candidate lists, then
//            topk_merge_kernel's merge, then the first n entries.  Entries past the row's non-NaN ones, and every entry of a
//            row with src == nullptr: UINT32_MAX and NaN.  A NaN in the row makes every logprob NaN, as it makes the score.
// ---------------------------------------------------------------------------------------
struct ScoreTopParams {
    const ScoreRow* rows;
    int V, nseg, top_n;
    float* cand_x;              // [rows of the launch][nseg][128]
    unsigned* cand_id;
    unsigned* out_id;           // [scored tokens][top_n]: row b's list at rows[b].dst
    float* out_lp;
};

__global__ void __launch_bounds__(TOPK_SEG_THREADS) score_top_segment_kernel(const __grid_constant__ ScoreTopParams p) {
    __shared__ float sx[TOPK_SEG];
    __shared__ unsigned sid[TOPK_SEG];
    const int seg = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    const float* src = p.rows[row].src;
    if (src == nullptr) return;
    const int seg0 = seg * TOPK_SEG;
#pragma unroll
    for (int j = 0; j < TOPK_SEG / TOPK_SEG_THREADS; ++j) {
        const int li = tid + TOPK_SEG_THREADS * j, i = seg0 + li;
        const float x = (i < p.V) ? __ldcg(src + i) : -INFINITY;
        const bool ranked = i < p.V && x == x;
        sx[li] = ranked ? x : -INFINITY;
        sid[li] = ranked ? (unsigned)i : 0xFFFFFFFFu;
    }
    sort_segment(sx, sid);
    __syncthreads();
    if (tid < TOPK_MAX) {
        const size_t o = ((size_t)row * p.nseg + seg) * TOPK_MAX + tid;
        p.cand_x[o] = sx[tid];
        p.cand_id[o] = sid[tid];
    }
}

__global__ void __launch_bounds__(TOPK_MERGE_THREADS) score_top_merge_kernel(const __grid_constant__ ScoreTopParams p) {
    __shared__ float sx[TOPK_MAX_SEGS * TOPK_MAX];
    __shared__ unsigned sid[TOPK_MAX_SEGS * TOPK_MAX];
    __shared__ ScoreAcc red[SCORE_THREADS / 32];
    __shared__ float s_m, s_log;
    __shared__ int s_nan;
    const int row = blockIdx.x, tid = threadIdx.x;
    const ScoreRow rw = p.rows[row];
    unsigned* oid = p.out_id + (size_t)rw.dst * p.top_n;
    float* olp = p.out_lp + (size_t)rw.dst * p.top_n;
    if (rw.src == nullptr) {
        if (tid < p.top_n) { oid[tid] = 0xFFFFFFFFu; olp[tid] = __int_as_float(0x7fc00000); }
        return;
    }
    if (tid < SCORE_THREADS) {
        ScoreAcc a{-INFINITY, 0.f, -INFINITY, 0xFFFFFFFFu, 0};
        score_row_warp(a, rw.src, p.V, tid);
        if ((tid & 31) == 0) red[tid >> 5] = a;
    } else {
        for (int i = tid - SCORE_THREADS; i < TOPK_MAX_SEGS * TOPK_MAX; i += TOPK_MERGE_THREADS - SCORE_THREADS) {
            const int sg = i / TOPK_MAX;
            const bool ok = sg < p.nseg;
            const size_t o = ((size_t)row * p.nseg + sg) * TOPK_MAX + (i % TOPK_MAX);
            sx[i] = ok ? p.cand_x[o] : -INFINITY;
            sid[i] = ok ? p.cand_id[o] : 0xFFFFFFFFu;
        }
    }
    __syncthreads();
    if (tid < 32) {
        ScoreAcc a;
        score_row_combine(a, red, tid);
        if (tid == 0) { s_m = a.m; s_log = logf(a.s); s_nan = a.nan; }
    }
    merge_lists(sx, sid);
    __syncthreads();
    if (tid < p.top_n) {
        const unsigned id = sid[tid];
        oid[tid] = id;
        olp[tid] = (s_nan || id == 0xFFFFFFFFu) ? __int_as_float(0x7fc00000) : (sx[tid] - s_m) - s_log;
    }
}

}  // namespace b200
