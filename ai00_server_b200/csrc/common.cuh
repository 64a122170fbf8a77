// Device-side helpers shared by all kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// ---------------------------------------------------------------------------------------
// Per-step metadata, one flat int array in HBM (rewritten by a single H2D copy per step so
// the captured CUDA graph never changes).  Layout: header, then arrays sized by the
// engine's token_chunk (maxT) and max_batch (maxS).
// ---------------------------------------------------------------------------------------
struct MetaView {
    const int* base;
    int maxT, maxS;
    __host__ __device__ int T() const { return base[0]; }        // tokens this step
    __host__ __device__ int nslots() const { return base[1]; }   // active slots this step
    __host__ __device__ int R() const { return base[2]; }        // logits rows this step
    __host__ __device__ const int* tok() const { return base + 8; }                       // [maxT] token ids
    __host__ __device__ const int* tok_slot() const { return base + 8 + maxT; }           // [maxT] state slot of token
    __host__ __device__ const int* tok_prev() const { return base + 8 + 2 * maxT; }       // [maxT] t-1 or -1 (take shift state)
    __host__ __device__ const int* tok_last() const { return base + 8 + 3 * maxT; }       // [maxT] 1 if last token of its slot in this step
    __host__ __device__ const int* out_tok() const { return base + 8 + 4 * maxT; }        // [maxT] logits row r -> token index
    __host__ __device__ const int* tok_outrow() const { return base + 8 + 5 * maxT; }     // [maxT] token -> logits row or -1
    __host__ __device__ const int* slot_id() const { return base + 8 + 6 * maxT; }        // [maxS] active slot -> state slot
    __host__ __device__ const int* slot_start() const { return base + 8 + 6 * maxT + maxS; }
    __host__ __device__ const int* slot_count() const { return base + 8 + 6 * maxT + 2 * maxS; }
    __host__ __device__ static size_t ints(int maxT, int maxS) { return 8 + 6 * (size_t)maxT + 3 * (size_t)maxS; }
};

// ---------------------------------------------------------------------------------------
// "A16" activation layout: the f16 operand of every projection, stored so that (a) the slice a GEMM stage needs -- one
// 128-wide k block of ALL tokens of the step -- is ONE contiguous run (one bulk TMA copy) and (b) that run IS the wgmma
// canonical K-major / no-swizzle B operand of `th` token rows, which ONE wgmma with N = th consumes:
//   [k block (128 k)][k8 chunk 16][th token rows][8 halves]      (8 rows x 16 B = one 128-byte core matrix)
// th = 16 x (token tiles of the step) = 16 / 32 / 64 / 128; a step's producers and consumers agree on it (the engine passes
// it to every launch).  One wide MMA per k step instead of one N = 16 MMA per token tile keeps the MMA issue count of a
// stage independent of the step's token count.
// Split operands (precision 1): th = 32, rows 0-15 hold the hi halves of the 16 tokens, rows 16-31 the lo halves.
// Every buffer reserves 128 token rows per k block and K padded to whole k blocks (padding k is multiplied by zero weights).
// ---------------------------------------------------------------------------------------
constexpr int A16_MAX_ROWS = 128;                      // token rows per k block: steps of up to 128 tokens
constexpr int A16_KB_HALVES = A16_MAX_ROWS * 128;      // halves per k block of a buffer
__host__ __device__ inline size_t a16_index(int m, int k, int th) {
    return (size_t)(k >> 7) * A16_KB_HALVES + ((size_t)((k >> 3) & 15) * th + m) * 8 + (k & 7);
}

__device__ __forceinline__ __half f2h_sat(float v) {
    v = fminf(fmaxf(v, -65504.f), 65504.f);
    return __float2half_rn(v);
}
// Split operand (precision 1 = f32 activations, DESIGN.md §2): a projection input v travels as two f16 numbers hi + lo = v
// (to ~2^-22 relative); hi sits at token row t, lo at row t + 16 of the same A16 buffer (the second 16-token tile), the
// projection multiplies both tiles and its epilogue adds the two accumulator tiles.
// Above |v| = 65504 hi saturates and lo carries the rest; lo saturates as well, so that a finite v never becomes an infinite
// operand: the pair saturates at +-131008 as the f16 operand does at +-65504.  NaN stays NaN in lo.
__device__ __forceinline__ void split_h(const float v, __half& hi, __half& lo) {
    hi = f2h_sat(v);
    const float rest = v - __half2float(hi);
    lo = __float2half_rn(fabsf(rest) > 65504.f ? copysignf(65504.f, rest) : rest);
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __halves2half2(f2h_sat(a), f2h_sat(b));
    return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ void split_pack_h2(const float a, const float b, uint32_t& hi, uint32_t& lo) {
    __half ah, al, bh, bl;
    split_h(a, ah, al);
    split_h(b, bh, bl);
    __half2 h = __halves2half2(ah, bh), l = __halves2half2(al, bl);
    hi = *reinterpret_cast<uint32_t*>(&h);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

// ---------------------------------------------------------------------------------------
// mbarrier + 1-D bulk TMA (cp.async.bulk -> SASS UBLKCP)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// ---------------------------------------------------------------------------------------
// Watchdog: every spin-wait in this library gives up after ~2 s, writes a record to mapped pinned
// host memory (so it survives the dead context) and traps: a protocol bug becomes a CUDA error
// with a diagnosis instead of a hung GPU.  g_watchdog is set once per process by the host.
// record: [0]=0xDEAD0000|code [1]=blockIdx.x [2]=threadIdx.x [3]=arg0 [4]=arg1 [5]=arg2
// ---------------------------------------------------------------------------------------
__device__ unsigned* g_watchdog = nullptr;
constexpr unsigned long long WATCHDOG_NS = 2000000000ull;
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __noinline__ void watchdog_fire(unsigned code, unsigned a0, unsigned a1, unsigned a2) {
    unsigned* w = g_watchdog;
    if (w) {
        w[1] = blockIdx.x; w[2] = threadIdx.x; w[3] = a0; w[4] = a1; w[5] = a2;
        __threadfence_system();
        w[0] = 0xDEAD0000u | code;
        __threadfence_system();
    }
    __trap();
}
struct SpinGuard {          // poll(): call once per spin iteration
    unsigned n = 0;
    unsigned long long t0 = 0;
    __device__ __forceinline__ void poll(unsigned code, unsigned a0, unsigned a1, unsigned a2) {
        if ((++n & 0x3FFu) == 0) {
            const unsigned long long t = globaltimer_ns();
            if (t0 == 0) t0 = t;
            else if (t - t0 > ((code == 2u || code == 3u) ? 2 * WATCHDOG_NS : WATCHDOG_NS)) watchdog_fire(code, a0, a1, a2);   // passive waiters (grid barrier, phase start) wait longest: the culprit reports first
        }
    }
};
enum WatchCode : unsigned { WD_MBAR = 1, WD_GRIDBAR = 2 };

__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// `tag` identifies the call site in watchdog reports
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, unsigned tag = 0) {
    if (mbar_try(bar, parity)) return;
    SpinGuard g;
    while (!mbar_try(bar, parity)) g.poll(WD_MBAR, bar, parity, tag);
}
// L2 policy for streamed-once weights
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar,
                                              uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            dst),
        "l"(src), "r"(bytes), "r"(bar), "l"(policy)
        : "memory");
}
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// fire-and-forget arrival: no value comes back, so the arriving thread pays a one-way trip
__device__ __forceinline__ void red_add_release_gpu(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_add_acq_rel_gpu(unsigned* p, unsigned v) {
    unsigned old;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu(unsigned* p, unsigned v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// D[16x8] += A[16x16] * B[16x8], f16 operands, f32 accumulate (legacy tensor path: HMMA)
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): the four warps of a warpgroup issue one m64nNk16 MMA together, both operands read
// from shared memory through matrix descriptors, the f32 accumulator in registers.  SASS: HGMMA.
// Accumulator fragment of m64nN: thread t of the warpgroup holds d[i], i < N/2, at row 16 (t / 32) + (t % 32) / 4 +
// 8 ((i % 4) / 2) and column 8 (i / 4) + 2 (t % 4) + (i % 2).
// ---------------------------------------------------------------------------------------
// shared-memory matrix descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes (128 B contiguous);
// lbo = byte distance between the two 16-byte k chunks of one k16 step, sbo = byte distance between 8-row groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// orders the warpgroup's register accesses (accumulator zeroing, epilogue reads) before the MMAs that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed MMA groups of this warp are still running
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x N] += A[64 x 16] * B[N x 16]^T, f16 operands (both K-major) -> f32, D in registers
template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b));
    }
};
template <>
struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b));
    }
};
template <>
struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b));
    }
};
template <>
struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b));
    }
};
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc) {
    Wgmma<N>::mma(d, a_desc, b_desc);
}

// Programmatic dependent launch: everything before griddepcontrol.wait may overlap the tail of the preceding kernel in the
// stream / graph (weights and step metadata are immutable while a step runs, so prefetching them may).
// profiling aid: globaltimer stamp i of this launch's trace row (CTA 0, thread 0 only; `tr` is null in production)
__device__ __forceinline__ void trace_stamp(unsigned long long* tr, const int i) {
    if (tr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        tr[i] = t;
    }
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// block-wide sum over 256 threads; `red` is >= 8 floats of shared memory; result broadcast
constexpr int CONSUMER_THREADS = 256;
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();   // protect `red` from the previous use
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < CONSUMER_THREADS / 32) ? red[lane] : 0.f;
    t = warp_sum(t);
    return t;
}
// generic versions for kernels with other block sizes (softmax)
__device__ __forceinline__ float block_sum_any(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < nw) ? red[lane] : 0.f;
    t = warp_sum(t);
    return t;
}
__device__ __forceinline__ float block_max_any(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < nw) ? red[lane] : -INFINITY;
    t = warp_max(t);
    return t;
}

// ---------------------------------------------------------------------------------------
// activations (exact-ish: expf/tanhf, not the fast intrinsics, to stay inside the 1e-3 budget)
// ---------------------------------------------------------------------------------------
enum Act : int { ACT_NONE = 0, ACT_TANH, ACT_SIGMOID, ACT_SILU, ACT_RELU2, ACT_EXPNEGEXP, ACT_V7DECAY };

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case ACT_TANH: return tanhf(v);
        case ACT_SIGMOID: return sigmoidf_(v);
        case ACT_SILU: return v * sigmoidf_(v);
        case ACT_RELU2: { float r = fmaxf(v, 0.f); return r * r; }
        case ACT_EXPNEGEXP: return expf(-expf(v));                       // v6 decay
        case ACT_V7DECAY: return expf(-0.606531f * sigmoidf_(v));        // v7 decay, exp(-0.5)
        default: return v;
    }
}

}  // namespace b200
