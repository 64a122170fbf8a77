// Softmax over the vocabulary, state layout transforms, small conversion kernels.
#pragma once
#include "common.cuh"

#include <cuda_bf16.h>

#include <type_traits>

namespace b200 {

// ---------------------------------------------------------------------------------------
// Row softmax (replaces `web_rwkv::runtime::softmax::softmax`, reference run.rs:1179).
// One CTA per row; the row (256 KB at V = 65536) is read twice from L2 and written once.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) softmax_kernel(const float* __restrict__ in, float* __restrict__ out, int V) {
    __shared__ float red[32];
    const float* x = in + (size_t)blockIdx.x * V;
    float* y = out + (size_t)blockIdx.x * V;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < V; i += blockDim.x) mx = fmaxf(mx, x[i]);
    mx = block_max_any(mx, red);
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(x[i] - mx);
    s = block_sum_any(s, red);
    const float inv = 1.0f / s;
    for (int i = threadIdx.x; i < V; i += blockDim.x) y[i] = expf(x[i] - mx) * inv;
}

// ---------------------------------------------------------------------------------------
// State import / export between the API layout and the device layout.
// API (web-rwkv shape [C, N+2, L, 1], x fastest; reference run.rs:987, lib.rs:267-272;
// SURVEY.md App. C) per slot: api[l][row][c], row 0 = time-mix shift, rows 1..N = WKV with
// row 1+i, col h*N+j <-> S[l,h][i][j], row N+1 = channel-mix shift.
// Device: att_shift[l][slot][c], ffn_shift[l][slot][c], wkv[l][slot][h][value][key].
// v5/v6: S[i=key][j=value]  -> M[value=j][key=i]   (transpose)
// v7:    S[i=value][j=key]  -> M[value=i][key=j]
// `h0`/`Hl`: first global head and head count held by this rank (tensor parallel).
// ---------------------------------------------------------------------------------------
struct StateXform {
    float* api;          // [L][N+2][C] staging in HBM
    // device side, addressed as base + l * layer_stride: a slot of the live state arrays or a snapshot record
    float* att; size_t att_ls;     // [C] per layer
    float* ffn; size_t ffn_ls;     // [C] per layer
    float* wkv; size_t wkv_ls;     // [Hl][64][64] per layer
    int L, C, Hl, h0, transpose;
};

template <bool IMPORT>
__global__ void state_xform_kernel(const StateXform p) {
    const int N = 64;
    const size_t per_layer = (size_t)(N + 2) * p.C;
    const size_t total = (size_t)p.L * per_layer;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int l = (int)(i / per_layer);
        const size_t r = i - (size_t)l * per_layer;
        const int row = (int)(r / p.C);
        const int c = (int)(r - (size_t)row * p.C);
        float* dev;
        if (row == 0) dev = p.att + (size_t)l * p.att_ls + c;
        else if (row == N + 1) dev = p.ffn + (size_t)l * p.ffn_ls + c;
        else {
            const int hg = c / N, j = c % N, ii = row - 1;
            const int hl = hg - p.h0;
            if (hl < 0 || hl >= p.Hl) {
                if (!IMPORT) p.api[i] = 0.f;
                continue;
            }
            const int val = p.transpose ? j : ii, key = p.transpose ? ii : j;
            dev = p.wkv + (size_t)l * p.wkv_ls + ((size_t)hl * N + val) * N + key;
        }
        if (IMPORT) *dev = p.api[i];
        else p.api[i] = *dev;
    }
}

// ---------------------------------------------------------------------------------------
// Tensor-parallel rendezvous: one flag word per (reader rank, writer rank) in the reader's comm
// block, written over NVLink peer memory.  The row-parallel projections leave their partial sums
// in the local comm block; after this barrier every rank's LN stage reads all ranks' partials
// straight from peer memory (one-shot all-reduce fused into the consumer, fixed rank order).
// The epoch lives in device memory so a captured graph replays correctly.
// ---------------------------------------------------------------------------------------
struct TpBar {
    unsigned* flags[8];     // flags[q]: rank q's flag array [8] (peer-mapped for q != rank)
    unsigned* epoch;        // local
    int rank, world;
};
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// threads 0..world-1 of one warp; all prior writes of the calling grid/CTA must already be ordered
// before the call (kernel boundary, or grid barrier + fence)
__device__ __forceinline__ void tp_barrier(const TpBar& b, const int lane) {
    unsigned e = 0;
    if (lane == 0) {
        e = *b.epoch + 1;
        *b.epoch = e;
    }
    e = __shfl_sync(0xffffffffu, e, 0);
    if (lane < b.world) {
        __threadfence_system();
        st_release_sys(b.flags[lane] + b.rank, e);
        SpinGuard sg_;
        while ((int)(ld_acquire_sys(b.flags[b.rank] + lane) - e) < 0) sg_.poll(5u, (unsigned)lane, e, (unsigned)b.rank);   // wrap-safe: epochs are 32-bit and only grow
    }
    __syncwarp();
    __threadfence_system();
}
__global__ void tp_barrier_kernel(const TpBar b) {
    // let the consumer (LN / front-half kernel) become resident and stage its static operands now: without this trigger it
    // is launched only when this kernel exits, and its launch + staging latency lands on every rendezvous
    pdl_launch_dependents();
    pdl_wait();
    tp_barrier(b, threadIdx.x);
}

// ---------------------------------------------------------------------------------------
// LoRA blend at load (reference lib.rs:466-485: `ModelBuilder::lora(Lora { data, blend: LoraBlend::full(alpha) })`):
//   W[o][i] <- f16( f32(W[o][i]) + alpha * sum_r B[o][r] * At[i][r] )
// with the on-disk layout the reference's converter writes (assets/scripts/convert_safetensors.py:96-101,
// crates/converter/src/main.rs:8-22): `<name>.lora.1` = lora_B [out, r], `<name>.lora.0` = lora_A transposed = [in, r].
// One thread per element, f32 accumulation in rank order, one rounding.
// ---------------------------------------------------------------------------------------
__global__ void lora_blend_kernel(__half* __restrict__ W, const __half* __restrict__ B, const __half* __restrict__ At, int out, int in,
                                  int r, float alpha) {
    const size_t n = (size_t)out * in;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const int o = (int)(e / in), i = (int)(e - (size_t)o * in);
        const __half* b = B + (size_t)o * r;
        const __half* a = At + (size_t)i * r;
        float acc = 0.f;
        for (int k = 0; k < r; ++k) acc = fmaf(__half2float(b[k]), __half2float(a[k]), acc);
        W[e] = __float2half_rn(__half2float(W[e]) + alpha * acc);
    }
}

__global__ void f16_to_f32_kernel(const __half* __restrict__ src, float* __restrict__ dst, size_t n, float scale, float bias) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = __half2float(src[i]) * scale + bias;
}

// f32 rows [T][K] -> a projection operand in the A16 layout of `th` token rows (b200rwkv_op_gemm): f16 rounding, or with `split`
// the hi / lo pair of common.cuh (hi at row t, lo at row t + 16).  Rows >= T and k >= K are left as they are.
__global__ void a16_from_f32_kernel(const float* __restrict__ src, int T, int K, int th, bool split, __half* __restrict__ dst) {
    const size_t n = (size_t)T * K;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int t = (int)(i / K), k = (int)(i - (size_t)t * K);
        if (split) split_h(src[i], dst[a16_index(t, k, th)], dst[a16_index(t + 16, k, th)]);
        else dst[a16_index(t, k, th)] = f2h_sat(src[i]);
    }
}

// BF16 or F32 weights handed over on the device (b200rwkv_update_weights_device) -> the F16 the build reads, rounded to nearest
// even; BF16 widens to f32 exactly first
template <typename T>
__global__ void to_f16_kernel(const T* __restrict__ src, __half* __restrict__ dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if constexpr (std::is_same<T, float>::value) dst[i] = __float2half_rn(src[i]);
        else dst[i] = __float2half_rn(__bfloat162float(src[i]));
    }
}

// v5 static decay: w = exp(-exp(time_decay))
__global__ void decay_table_kernel(const __half* __restrict__ src, float* __restrict__ dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = expf(-expf(__half2float(src[i])));
}

// ---------------------------------------------------------------------------------------
// Pooled hidden rows (b200rwkv_keep_hidden_pooled): one [C] f32 row per entry of an infer call and pooled layer, reduced from
// the [T][C] step buffers the LN stages record the residual stream into, so the embeddings route moves num_emb floats per
// input to the host instead of every token's row.  One launch after every step of the call: CTA (entry of the step, pooled
// layer, block of POOL_THREADS float4 columns), one float4 column per thread.
//   POOL_LAST: dst <- the entry's last row of the step (a later step of the same entry overwrites it).
//   POOL_MEAN: acc = +0.0 on the entry's first step, else dst; acc = __fadd_rn(acc, row) for the step's rows in token order;
//              the step that holds the entry's final token of the call stores __fdiv_rn(acc, ntok), the others store acc.
// A channel's sum is one chain of adds in token order whatever the cut into steps, so the bits do not depend on the cut.
// The steps of a call run in order on one stream: the running sum needs no atomics.
// ---------------------------------------------------------------------------------------
struct PoolEntry {
    int row0, nrows;            // the entry's rows of this step: [row0, row0 + nrows) of the step buffers
    int dst;                    // destination row (the entry's index in the call)
    int pos, ntok;              // tokens of the entry before this step, and in the whole call
};
constexpr int POOL_MAX_LAYERS = 8;
constexpr int POOL_THREADS = 256;
struct PoolParams {
    const PoolEntry* ent;       // [gridDim.x]
    const float* src[POOL_MAX_LAYERS];      // step buffer [T][C] of pooled layer k
    float* dst;                 // [layers][dst_rows][C]
    int C, dst_rows, mode;      // mode: B200RWKV_POOL_LAST (0) / B200RWKV_POOL_MEAN (1)
};

__global__ void __launch_bounds__(POOL_THREADS) hidden_pool_kernel(const __grid_constant__ PoolParams p) {
    const int ld = p.C / 4, c4 = blockIdx.z * POOL_THREADS + threadIdx.x;
    if (c4 >= ld) return;
    const PoolEntry en = p.ent[blockIdx.x];
    const float4* src = reinterpret_cast<const float4*>(p.src[blockIdx.y]) + (size_t)en.row0 * ld + c4;
    float4* dst = reinterpret_cast<float4*>(p.dst) + ((size_t)blockIdx.y * p.dst_rows + en.dst) * ld + c4;
    if (p.mode == 0) {
        *dst = src[(size_t)(en.nrows - 1) * ld];
        return;
    }
    float4 a = en.pos == 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : *dst;
#pragma unroll 8
    for (int t = 0; t < en.nrows; ++t) {
        const float4 v = src[(size_t)t * ld];
        a.x = __fadd_rn(a.x, v.x); a.y = __fadd_rn(a.y, v.y); a.z = __fadd_rn(a.z, v.z); a.w = __fadd_rn(a.w, v.w);
    }
    if (en.pos + en.nrows == en.ntok) {
        const float n = (float)en.ntok;
        a.x = __fdiv_rn(a.x, n); a.y = __fdiv_rn(a.y, n); a.z = __fdiv_rn(a.z, n); a.w = __fdiv_rn(a.w, n);
    }
    *dst = a;
}

}  // namespace b200
