// Streaming micro-benchmarks (debug entry point b200rwkv_debug_stream): how fast can one GPU pull
// a large buffer from HBM through (a) plain vector loads, (b) the 1-D bulk-TMA stage ring used by
// the projection GEMM with a trivial consumer.
// Not on the product path; used to size the ring and to separate producer limits from consumer limits.
#pragma once
#include "gemm.cuh"

namespace b200 {

__global__ void __launch_bounds__(256) stream_ldg_kernel(const uint4* __restrict__ src, size_t n16, unsigned* sink) {
    unsigned acc = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 7 * stride < n16; i += 8 * stride) {
        uint4 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __ldcs(src + i + j * stride);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc ^= v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
    }
    if (acc == 0x12345u) *sink = acc;
}

struct StreamParams {
    const uint8_t* src;
    size_t bytes_per_cta;
    int stage_bytes;     // multiple of 1024
    int nstage;
    int use_hint;        // 0 none, 1 evict_first
    int split;           // bulk copies per stage (1, 2, 4)
    int producers;       // producer warps issuing in round robin (1..3)
    int extra;           // bytes of the stage sent as a separate small copy (the GEMM's activation slice)
};

// one CTA per SM, warp 0 lanes = producers, warp 1 lane 0 = consumer
__global__ void __launch_bounds__(128, 1) stream_ring_kernel(const __grid_constant__ StreamParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t smem_base = smem_u32(smem);
    const int NS = p.nstage, SB = p.stage_bytes;
    const uint32_t full_bar = smem_base + NS * SB;
    const uint32_t empty_bar = full_bar + NS * 8;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(full_bar + s * 8, 1); mbar_init(empty_bar + s * 8, 1); }
        mbar_fence_init();
    }
    __syncthreads();
    const size_t nst = p.bytes_per_cta / SB;
    const uint8_t* src = p.src + (size_t)blockIdx.x * p.bytes_per_cta;
    // producers: lane 0 of warps 0, 2, 3 (round robin over stages); consumer: lane 0 of warp 1
    const int prod_id = (warp == 0) ? 0 : (warp == 2 ? 1 : (warp == 3 ? 2 : -1));
    if (prod_id >= 0 && prod_id < p.producers && lane == 0) {
        const uint64_t pol = l2_policy_evict_first();
        const int piece = (SB - p.extra) / p.split;
        int stage = prod_id;
        uint32_t par = 1;                 // parity of the previous use
        while (stage >= NS) { stage -= NS; par ^= 1u; }
        unsigned seq = prod_id;
        for (size_t it = prod_id; it < nst; it += p.producers, seq += p.producers) {
            if (seq >= (unsigned)NS) mbar_wait(empty_bar + stage * 8, par);
            mbar_expect_tx(full_bar + stage * 8, SB);
            const uint8_t* g = src + it * (size_t)SB;
            for (int s_ = 0; s_ < p.split; ++s_) {
                if (p.use_hint) bulk_g2s_hint(smem_base + stage * SB + s_ * piece, g + (size_t)s_ * piece, piece, full_bar + stage * 8, pol);
                else bulk_g2s(smem_base + stage * SB + s_ * piece, g + (size_t)s_ * piece, piece, full_bar + stage * 8);
            }
            if (p.extra) bulk_g2s(smem_base + stage * SB + (SB - p.extra), g + (SB - p.extra), p.extra, full_bar + stage * 8);
            stage += p.producers;
            while (stage >= NS) { stage -= NS; par ^= 1u; }
        }
    } else if (warp == 1 && lane == 0) {
        int stage = 0;
        uint32_t par = 0;
        for (size_t it = 0; it < nst; ++it) {
            mbar_wait(full_bar + stage * 8, par);
            mbar_arrive(empty_bar + stage * 8);
            if (++stage == NS) { stage = 0; par ^= 1u; }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------
// L2 prefetch micro-benchmark (b200rwkv_debug_prefetch): does a prefetch issued while HBM is IDLE make the next streaming
// launch faster?  Kernel P: CTA i asks L2 for `nblk` 32 KB blocks of the range consumer CTA i will stream (after its first
// `skip` blocks), then idles `idle_ns`; kernel S = stream_ring_kernel over the same buffer.  mode 0: one thread, bulk
// prefetches; 1: the 32 lanes of warp 0 issue them round robin; 2: every thread issues 128-byte prefetch.global.L2.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) prefetch_probe_kernel(const uint8_t* src, size_t bytes_per_cta, int consumers, int skip,
                                                             int nblk, int mode, unsigned long long idle_ns) {
    const unsigned long long t0 = globaltimer_ns();
    for (int c = blockIdx.x; c < consumers; c += gridDim.x) {
        const uint8_t* base = src + (size_t)c * bytes_per_cta + (size_t)skip * 32768;
        const size_t avail = bytes_per_cta > (size_t)skip * 32768 ? (bytes_per_cta - (size_t)skip * 32768) / 32768 : 0;
        const int n = (int)min((size_t)nblk, avail);
        if (mode == 0) {
            if (threadIdx.x == 0)
                for (int i = 0; i < n; ++i) bulk_prefetch_l2(base + (size_t)i * 32768, 32768);
        } else if (mode == 1) {
            if (threadIdx.x < 32)
                for (int i = threadIdx.x; i < n; i += 32) bulk_prefetch_l2(base + (size_t)i * 32768, 32768);
        } else {
            for (size_t off = (size_t)threadIdx.x * 128; off < (size_t)n * 32768; off += 128 * 128)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(base + off));
        }
    }
    while (globaltimer_ns() - t0 < idle_ns) { }
}

}  // namespace b200