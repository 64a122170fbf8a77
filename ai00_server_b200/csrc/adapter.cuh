// Unblended LoRA adapters (b200rwkv_create_adapters): the "shrink" half of a bound adapter's low-rank term.
//
// A projection W that some adapter touches has a second weight layout W' = [W | a_1 B_1 | ... | a_n B_n] (engine.cu, one
// zero-padded 128-wide k block per adapter after W's own k blocks), and its A16 operand buffer carries the same n tail
// blocks.  For every token row of a step, adapter_shrink_kernel computes u = x A_a^T in f32 for the adapter a its slot is
// bound to, from exactly the operand values the projection itself multiplies (f16, or the hi + lo pair), and stores u rounded
// to the operand format into tail block a; every other tail block of the row gets zeros.  The unchanged projection kernel then
// multiplies W' by [x | 0 .. u .. 0], which adds a_a B_a u before its epilogue's bias and activation.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int AD_MAX = 8;              // adapters per engine
constexpr int AD_MAX_RANK = 128;       // one k block of W' per adapter
constexpr int AD_MAX_PROJ = 4;         // projections one launch serves (R / K / V / G read the same step phase)
constexpr int AD_COLS = 8;             // columns j of u per CTA: 16 CTAs cover the 128 columns of a tail block
constexpr int AD_WARPS = 16;           // the CTA's warps split K (a decode launch is bound by load latency, not bytes)
constexpr int AD_THREADS = AD_WARPS * 32;
constexpr int AD_TOK = 16;             // token rows per CTA

struct AdapterProj {
    __half* op;                        // the projection's A16 operand buffer
    int K;                             // operand columns the projection reads; tail block b - 1 starts at k = kb0 * 128
    int kb0;
    const __half* A[AD_MAX];           // adapter b + 1: [r rounded up to 8][K] f16 (lora.0 transposed, zero rows past r), null: no pair
    int r[AD_MAX];
};

struct AdapterParams {
    AdapterProj p[AD_MAX_PROJ];
    int nproj, n;                      // projections, adapters
    MetaView meta;
    const int* slot_adapter;           // [S] adapter bound to each slot, 0 = none
    int head;                          // rows are the step's output rows (the head's operand), else its tokens
    int th;                            // A16 token rows of the operands (set per step)
};

// SPLIT: hi + lo operands (precision 1), rows 0-15 hi, 16-31 lo
template <bool SPLIT>
__global__ void __launch_bounds__(AD_THREADS) adapter_shrink_kernel(AdapterParams P) {
    pdl_launch_dependents();
    const AdapterProj& pr = P.p[blockIdx.z];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j0 = blockIdx.x * AD_COLS;
    const int m0 = blockIdx.y * AD_TOK;
    // the step's metadata and the binding table do not change while a step runs: read them before the wait
    const int nrows = P.head ? P.meta.R() : P.meta.T();
    __shared__ int s_ad[AD_TOK];
    __shared__ float s_part[AD_WARPS][AD_COLS][AD_TOK];
    if (threadIdx.x < AD_TOK) {
        const int m = m0 + threadIdx.x;
        int a = 0;
        if (m < nrows) {
            const int t = P.head ? P.meta.out_tok()[m] : m;
            a = P.slot_adapter[P.meta.tok_slot()[t]];
        }
        s_ad[threadIdx.x] = a;
    }
    __syncthreads();
    pdl_wait();
    if (m0 >= nrows) return;
    const int nm = min(AD_TOK, nrows - m0);
    auto has = [&](int a, int j) { return a > 0 && j < pr.r[a - 1] && pr.A[a - 1] != nullptr; };
    bool any = false;
    for (int i = 0; i < nm; ++i) any |= has(s_ad[i], j0);

    if (any) {
        // lane l works on row m0 + (l % 16); warp w takes the k8 chunks 2 w + l / 16 + 32 n, so the 32 lanes of one operand
        // load read two whole chunks of the 16 rows (512 contiguous bytes of the A16 layout), and lanes of one adapter share
        // their A loads
        const int i = lane & 15;
        const int a = s_ad[i];
        float acc[AD_COLS];
#pragma unroll
        for (int c = 0; c < AD_COLS; ++c) acc[c] = 0.f;
        if (i < nm && has(a, j0)) {
            // A holds whole groups of 8 rows (zeros past the rank), so every column of the CTA has a row: the loop body has no
            // branch, and the operand load and all eight A loads of an iteration (of two, unrolled) are in flight together
            const int K = pr.K, th = P.th;
            const __half* arow = pr.A[a - 1] + (size_t)j0 * K;
            const __half* op = pr.op;
#pragma unroll 2
            for (int k = (warp * 2 + (lane >> 4)) * 8; k < K; k += AD_WARPS * 16) {
                uint4 wa[AD_COLS];
#pragma unroll
                for (int c = 0; c < AD_COLS; ++c) wa[c] = __ldg(reinterpret_cast<const uint4*>(arow + (size_t)c * K + k));
                const uint4 xh = *reinterpret_cast<const uint4*>(op + a16_index(m0 + i, k, th));
                uint4 xl = make_uint4(0, 0, 0, 0);
                if (SPLIT) xl = *reinterpret_cast<const uint4*>(op + a16_index(m0 + i + 16, k, th));
                float xf[8];
                const __half2* x2 = reinterpret_cast<const __half2*>(&xh);
                const __half2* l2 = reinterpret_cast<const __half2*>(&xl);
#pragma unroll
                for (int q = 0; q < 4; ++q) {       // the hi + lo pair in f32; + 0 without split operands
                    const float2 h = __half22float2(x2[q]), l = __half22float2(l2[q]);
                    xf[2 * q] = h.x + l.x;
                    xf[2 * q + 1] = h.y + l.y;
                }
#pragma unroll
                for (int c = 0; c < AD_COLS; ++c) {
                    const __half2* w2 = reinterpret_cast<const __half2*>(&wa[c]);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float2 wf = __half22float2(w2[q]);
                        acc[c] = fmaf(xf[2 * q], wf.x, acc[c]);
                        acc[c] = fmaf(xf[2 * q + 1], wf.y, acc[c]);
                    }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < AD_COLS; ++c) {
            acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 16);
            if (lane < AD_TOK) s_part[warp][c][lane] = acc[c];
        }
    }
    __syncthreads();
    // thread (c, i) < 128: column j0 + c of row m0 + i in every tail block (and its lo row), the warps' partials summed in order
    if (threadIdx.x < AD_COLS * AD_TOK) {
        const int c = threadIdx.x / AD_TOK, i = threadIdx.x % AD_TOK, j = j0 + c;
        if (i < nm) {
            const int a = s_ad[i];
            __half hi = __float2half_rn(0.f), lo = hi;
            if (any && has(a, j)) {
                float u = 0.f;
                for (int w = 0; w < AD_WARPS; ++w) u += s_part[w][c][i];
                if (SPLIT) split_h(u, hi, lo);
                else hi = f2h_sat(u);
            }
            const __half zero = __float2half_rn(0.f);
            const int m = m0 + i;
            for (int b = 1; b <= P.n; ++b) {
                const int k = (pr.kb0 + b - 1) * 128 + j;
                pr.op[a16_index(m, k, P.th)] = b == a ? hi : zero;
                if (SPLIT) pr.op[a16_index(m + 16, k, P.th)] = b == a ? lo : zero;
            }
        }
    }
}

// one CTA per (8 columns of u, 16 rows, projection)
inline dim3 adapter_grid(int rows, int nproj) { return dim3(AD_MAX_RANK / AD_COLS, (rows + AD_TOK - 1) / AD_TOK, nproj); }

}  // namespace b200
