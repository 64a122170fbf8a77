// b200rwkv engine: model build from `.st`, per-step kernel schedule, state ops, C ABI.
// Host side is plain C++ (the reference's engine, web-rwkv, is compiled Rust; no Rust toolchain
// exists in this image) — see include/b200rwkv.h for the reference call site of every entry.
#include "../../include/b200rwkv.h"

#include <unistd.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <thread>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "gemm.cuh"
#include "qgemm.cuh"
#include "fp8gemm.cuh"
#include "int4gemm.cuh"
#include "pre6.cuh"
#include "sample.cuh"
#include "misc.cuh"
#include "mix.cuh"
#include "wkv.cuh"
#include "adapter.cuh"

namespace b200 {

// =========================================================================================
// errors
// =========================================================================================
struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
#define CK(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess)                                                                           \
            throw Error(B200RWKV_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_) + " @" +   \
                                               __FILE__ + ":" + std::to_string(__LINE__) + watchdog_report()); \
    } while (0)
#define REQUIRE(cond, code, msg)                 \
    do {                                         \
        if (!(cond)) throw Error((code), (msg)); \
    } while (0)

static thread_local std::string g_err;

// watchdog record in mapped pinned host memory (see common.cuh)
static unsigned* g_wd_host = nullptr;
static void watchdog_setup() {
    if (g_wd_host) { memset(g_wd_host, 0, 64); return; }
    unsigned* h = nullptr;
    if (cudaHostAlloc(&h, 64, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return;
    memset(h, 0, 64);
    g_wd_host = h;
}
static std::string watchdog_report() {
    if (!g_wd_host || (g_wd_host[0] >> 16) != 0xDEADu) return "";
    char buf[256];
    snprintf(buf, sizeof buf, " [device watchdog: code=%u block=%u thread=%u a0=0x%x a1=%u a2=%u]", g_wd_host[0] & 0xFFFFu, g_wd_host[1],
             g_wd_host[2], g_wd_host[3], g_wd_host[4], g_wd_host[5]);
    return buf;
}

// =========================================================================================
// owners of CUDA resources: move-only, released when they go out of scope (destructors ignore errors), and usable
// wherever the raw pointer or handle is
// =========================================================================================
// A device (cudaMalloc) or pinned host (cudaMallocHost) block of `bytes` bytes
template <typename T, bool Pinned = false>
struct Buf {
    T* p = nullptr;
    size_t bytes = 0;
    Buf() = default;
    explicit Buf(size_t n) { grow(n, n); }
    Buf(Buf&& o) noexcept : p(std::exchange(o.p, nullptr)), bytes(std::exchange(o.bytes, (size_t)0)) {}
    Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(bytes, o.bytes); return *this; }
    ~Buf() { if (p) Pinned ? cudaFreeHost(p) : cudaFree(p); }
    operator T*() const { return p; }
    // Smaller than `need` bytes: free the block, then allocate `alloc` bytes.  Freeing first keeps the peak at the new block;
    // a failed allocation leaves the owner empty, so the next call retries.
    void grow(size_t need, size_t alloc) {
        if (bytes >= need) return;
        T* old = std::exchange(p, nullptr);
        bytes = 0;
        if (old) CK(Pinned ? cudaFreeHost(old) : cudaFree(old));
        void* q = nullptr;
        CK(Pinned ? cudaMallocHost(&q, alloc) : cudaMalloc(&q, alloc));
        p = static_cast<T*>(q);
        bytes = alloc;
    }
};
template <typename T> using HostBuf = Buf<T, true>;

template <typename H, cudaError_t (*Destroy)(H)>
struct Handle {
    H h = nullptr;
    Handle() = default;
    explicit Handle(H x) : h(x) {}
    Handle(Handle&& o) noexcept : h(std::exchange(o.h, nullptr)) {}
    Handle& operator=(Handle&& o) noexcept { std::swap(h, o.h); return *this; }
    ~Handle() { if (h) Destroy(h); }
    operator H() const { return h; }
};
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using GraphExec = Handle<cudaGraphExec_t, cudaGraphExecDestroy>;

static Event new_event(unsigned flags = cudaEventDefault) {
    cudaEvent_t ev = nullptr;
    CK(cudaEventCreateWithFlags(&ev, flags));
    return Event(ev);
}
static Stream new_stream() {
    cudaStream_t s = nullptr;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return Stream(s);
}
// The work `enqueue` issues on `s`, captured into a graph and instantiated; a throw ends and drops the partial capture.
template <typename F>
static GraphExec capture_graph(cudaStream_t s, F&& enqueue) {
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    try {
        enqueue();
    } catch (...) {
        cudaStreamEndCapture(s, &g);
        if (g) cudaGraphDestroy(g);
        throw;
    }
    CK(cudaStreamEndCapture(s, &g));
    cudaGraphExec_t ge = nullptr;
    const cudaError_t instantiated = cudaGraphInstantiate(&ge, g, 0);
    cudaGraphDestroy(g);
    CK(instantiated);
    return GraphExec(ge);
}

// =========================================================================================
// safetensors reader (header = u64 LE length + JSON object; tensor bytes follow)
// =========================================================================================
struct StTensor {
    std::string name;
    std::string dtype;
    std::vector<int64_t> shape;
    const uint8_t* data = nullptr;
    size_t nbytes = 0;
    int64_t numel() const {
        int64_t n = 1;
        for (auto d : shape) n *= d;
        return n;
    }
};

class StFile {
public:
    std::map<std::string, StTensor> tensors;
    bool duplicate = false;     // the header names a tensor twice (`tensors` holds the first)

    StFile() {}           // tensors filled by the caller (b200rwkv_op_gemm_tail's tail columns)
    StFile(const uint8_t* buf, size_t len) {
        REQUIRE(buf && len >= 8, B200RWKV_ERR_INVALID, "safetensors: buffer too small");
        uint64_t hlen = 0;
        memcpy(&hlen, buf, 8);
        REQUIRE(hlen <= len - 8, B200RWKV_ERR_INVALID, "safetensors: bad header length");
        s_ = reinterpret_cast<const char*>(buf + 8);
        n_ = (size_t)hlen;
        i_ = 0;
        const uint8_t* base = buf + 8 + hlen;
        const size_t data_len = len - 8 - hlen;
        ws();
        expect('{');
        ws();
        if (peek() == '}') return;
        for (;;) {
            ws();
            std::string key = str();
            ws();
            expect(':');
            ws();
            if (key == "__metadata__") {
                skip_value();
            } else {
                StTensor t;
                size_t b = 0, e = 0;
                expect('{');
                for (;;) {
                    ws();
                    std::string k = str();
                    ws();
                    expect(':');
                    ws();
                    if (k == "dtype") t.dtype = str();
                    else if (k == "shape") {
                        auto v = int_array();
                        t.shape.assign(v.begin(), v.end());
                    } else if (k == "data_offsets") {
                        auto v = int_array();
                        REQUIRE(v.size() == 2, B200RWKV_ERR_INVALID, "safetensors: data_offsets");
                        b = (size_t)v[0];
                        e = (size_t)v[1];
                    } else skip_value();
                    ws();
                    if (peek() == ',') { ++i_; continue; }
                    expect('}');
                    break;
                }
                REQUIRE(b <= e && e <= data_len, B200RWKV_ERR_INVALID, "safetensors: tensor out of bounds: " + key);
                t.data = base + b;
                t.nbytes = e - b;
                // byte length must equal dtype size x shape product (overflow-checked): every later size check trusts numel()
                const size_t esz = dtype_size(t.dtype);
                REQUIRE(esz > 0, B200RWKV_ERR_INVALID, "safetensors: unknown dtype '" + t.dtype + "' of " + key);
                REQUIRE(t.shape.size() <= 8, B200RWKV_ERR_INVALID, "safetensors: too many dimensions: " + key);
                uint64_t ne = 1;
                for (int64_t d : t.shape) {
                    REQUIRE(d >= 0 && (d == 0 || ne <= (uint64_t)1 << 40) && (uint64_t)d <= ((uint64_t)1 << 40), B200RWKV_ERR_INVALID,
                            "safetensors: bad shape of " + key);
                    ne *= (uint64_t)d;
                }
                REQUIRE(ne <= ((uint64_t)1 << 44) && ne * esz == (uint64_t)t.nbytes, B200RWKV_ERR_INVALID,
                        "safetensors: byte length of " + key + " does not match dtype x shape");
                t.name = key;
                if (!tensors.emplace(std::move(key), std::move(t)).second) duplicate = true;
            }
            ws();
            if (peek() == ',') { ++i_; continue; }
            expect('}');
            break;
        }
    }
    const StTensor* find(const std::string& name) const {
        auto it = tensors.find(name);
        return it == tensors.end() ? nullptr : &it->second;
    }
    const StTensor& get(const std::string& name) const {
        auto* t = find(name);
        REQUIRE(t, B200RWKV_ERR_INVALID, "missing tensor: " + name);
        REQUIRE(t->dtype == "F16", B200RWKV_ERR_UNSUPPORTED, "tensor " + name + " is " + t->dtype + ", expected F16");
        return *t;
    }

    static size_t dtype_size(const std::string& d) {
        if (d == "F16" || d == "BF16" || d == "I16" || d == "U16") return 2;
        if (d == "F32" || d == "I32" || d == "U32") return 4;
        if (d == "F64" || d == "I64" || d == "U64") return 8;
        if (d == "I8" || d == "U8" || d == "BOOL" || d == "F8_E4M3" || d == "F8_E5M2") return 1;
        return 0;
    }
    // dimension i of a tensor that must have exactly `rank` dimensions (0 = any rank > i)
    static int64_t dim(const StTensor& t, size_t i, const std::string& name, size_t rank = 0) {
        REQUIRE((rank == 0 || t.shape.size() == rank) && i < t.shape.size(), B200RWKV_ERR_INVALID, "unexpected rank of tensor " + name);
        REQUIRE(t.shape[i] > 0 && t.shape[i] <= (int64_t)1 << 30, B200RWKV_ERR_INVALID, "bad dimension of tensor " + name);
        return t.shape[i];
    }
    int64_t dim(const std::string& name, size_t i, size_t rank = 0) const { return dim(get(name), i, name, rank); }

private:
    const char* s_;
    size_t n_, i_;
    int depth_ = 0;
    char peek() { return i_ < n_ ? s_[i_] : '\0'; }
    void ws() { while (i_ < n_ && (s_[i_] == ' ' || s_[i_] == '\n' || s_[i_] == '\t' || s_[i_] == '\r')) ++i_; }
    void expect(char c) {
        REQUIRE(peek() == c, B200RWKV_ERR_INVALID, std::string("safetensors: expected '") + c + "'");
        ++i_;
    }
    std::string str() {
        expect('"');
        std::string out;
        while (i_ < n_ && s_[i_] != '"') {
            if (s_[i_] == '\\' && i_ + 1 < n_) {
                ++i_;
                char c = s_[i_];
                if (c == 'n') out.push_back('\n');
                else if (c == 't') out.push_back('\t');
                else if (c == 'u') { i_ += 4; out.push_back('?'); }
                else out.push_back(c);
            } else out.push_back(s_[i_]);
            ++i_;
        }
        expect('"');
        return out;
    }
    std::vector<int64_t> int_array() {
        std::vector<int64_t> v;
        expect('[');
        ws();
        if (peek() == ']') { ++i_; return v; }
        for (;;) {
            ws();
            int64_t x = 0;
            bool any = false;
            while (i_ < n_ && s_[i_] >= '0' && s_[i_] <= '9') { x = x * 10 + (s_[i_] - '0'); ++i_; any = true; }
            REQUIRE(any, B200RWKV_ERR_INVALID, "safetensors: expected integer");
            v.push_back(x);
            ws();
            if (peek() == ',') { ++i_; continue; }
            expect(']');
            break;
        }
        return v;
    }
    struct DepthGuard {
        int& d;
        explicit DepthGuard(int& d_) : d(d_) { ++d; }
        ~DepthGuard() { --d; }
    };
    void skip_value() {
        DepthGuard dg(depth_);
        REQUIRE(depth_ <= 64, B200RWKV_ERR_INVALID, "safetensors: header nested too deeply");
        ws();
        char c = peek();
        if (c == '"') { (void)str(); return; }
        if (c == '{' || c == '[') {
            const char close = (c == '{') ? '}' : ']';
            ++i_;
            ws();
            if (peek() == close) { ++i_; return; }
            for (;;) {
                ws();
                if (c == '{') { (void)str(); ws(); expect(':'); }
                skip_value();
                ws();
                if (peek() == ',') { ++i_; continue; }
                expect(close);
                return;
            }
        }
        while (i_ < n_ && s_[i_] != ',' && s_[i_] != '}' && s_[i_] != ']') ++i_;
    }
};

// Mirror of web-rwkv `Loader::info` (reference lib.rs:587): version and dims from names/shapes.
static b200rwkv_info derive_info(const StFile& st) {
    b200rwkv_info o;
    memset(&o, 0, sizeof(o));
    o.num_vocab = (int)st.dim("emb.weight", 0, 2);
    o.num_emb = (int)st.dim("emb.weight", 1, 2);
    int L = 0;
    while (st.find("blocks." + std::to_string(L) + ".ln1.weight")) ++L;
    REQUIRE(L > 0, B200RWKV_ERR_INVALID, "no blocks.*.ln1.weight tensors");
    o.num_layer = L;
    o.num_hidden = (int)st.dim("blocks.0.ffn.key.weight", 0, 2);
    if (st.find("blocks.0.att.r_k")) {
        o.version = 7;
        o.num_head = (int)st.dim("blocks.0.att.r_k", 0, 2);
        o.head_size = (int)st.dim("blocks.0.att.r_k", 1, 2);
        o.time_decay_adapter = (int)st.dim("blocks.0.att.w1", 0, 2);
    } else if (st.find("blocks.0.att.time_mix_w1")) {
        o.version = 6;
        o.num_head = (int)st.dim("blocks.0.att.time_first", 0, 2);
        o.head_size = (int)st.dim("blocks.0.att.time_first", 1, 2);
        o.time_mix_adapter = (int)st.dim("blocks.0.att.time_mix_w1", 0, 2) / 5;
        o.time_decay_adapter = (int)st.dim("blocks.0.att.time_decay_w1", 0, 2);
    } else if (st.find("blocks.0.att.ln_x.weight") && st.find("blocks.0.att.gate.weight")) {
        o.version = 5;
        REQUIRE(st.get("blocks.0.att.time_first").shape.size() == 2, B200RWKV_ERR_UNSUPPORTED, "v5.0 (scalar time_first) is not supported");
        o.num_head = (int)st.dim("blocks.0.att.time_first", 0, 2);
        o.head_size = (int)st.dim("blocks.0.att.time_first", 1, 2);
    } else {
        throw Error(B200RWKV_ERR_UNSUPPORTED, "unsupported model version (RWKV v5.1/5.2, v6, v7 are supported)");
    }
    return o;
}

static float st_elem_f32(const StTensor& t, size_t i) {
    if (t.dtype == "F16") return __half2float(reinterpret_cast<const __half*>(t.data)[i]);
    if (t.dtype == "F32") { float v; memcpy(&v, t.data + i * 4, 4); return v; }
    if (t.dtype == "BF16") { uint32_t u = (uint32_t)reinterpret_cast<const uint16_t*>(t.data)[i] << 16; float v; memcpy(&v, &u, 4); return v; }
    throw Error(B200RWKV_ERR_UNSUPPORTED, "tensor " + t.name + " is " + t.dtype + ", expected F16 / F32 / BF16");
}

// `vN::read_state` (reference lib.rs:378-389) and `State::init` with a state-tuned model (run.rs:477, lib.rs:452-462):
// `blocks.{l}.att.time_state` [H, N, N] (transposed by the converter, convert_safetensors.py:101, crates/converter/src/main.rs:20)
// -> the host state tensor [L][N+2][C]: row 1+i, column h*N+j <- time_state[h][i][j]; shift rows zero.
// Returns false (and leaves `out` empty) when the file carries no time_state.
static void time_state_rows(const StTensor& ts, int l, int H, int N, int C, std::vector<float>& out) {
    for (int h = 0; h < H; ++h)
        for (int i = 0; i < N; ++i)
            for (int j = 0; j < N; ++j)
                out[((size_t)l * (N + 2) + 1 + i) * C + h * N + j] = st_elem_f32(ts, ((size_t)h * N + i) * N + j);
}
static bool state_from_st(const StFile& st, int L, int H, int N, int C, std::vector<float>& out) {
    if (!st.find("blocks.0.att.time_state")) return false;
    out.assign((size_t)L * (N + 2) * C, 0.f);
    for (int l = 0; l < L; ++l) {
        const std::string name = "blocks." + std::to_string(l) + ".att.time_state";
        const StTensor* ts = st.find(name);
        REQUIRE(ts, B200RWKV_ERR_INVALID, "missing tensor: " + name);
        REQUIRE(ts->numel() == (int64_t)H * N * N, B200RWKV_ERR_INVALID, "time_state must be [num_head, head_size, head_size]: " + name);
        (void)st_elem_f32(*ts, 0);          // the dtype: F16, F32 or BF16
        time_state_rows(*ts, l, H, N, C, out);
    }
    return true;
}

// =========================================================================================
// engine
// =========================================================================================
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

enum KClass { KC_GEMM = 0, KC_WKV = 1, KC_LN = 2, KC_OTHER = 3 };

struct SegDesc {
    const StTensor* t = nullptr;
    int64_t slice = -1;        // leading-dim index for 3-D tensors
    int n0 = 0, N = 0, k0 = 0, K = 0;
    GemmSeg proto;             // A, out_mode, act, bias, out, ldo, grp, grp_stride, aux*
    int ad_tail = 0;           // unblended adapters: 128-wide tail k blocks after the segment's own (make_launch)
    SegDesc() { memset(&proto, 0, sizeof(proto)); }
};

// One weight fill of the build: the tensor it reads (the key of b200rwkv_engine::fills), what it makes of it and where that
// goes.  The build records the fills while it plans; b200rwkv_engine::fill_weights runs them, once at creation and again
// for every tensor a weight update lists, so an update writes exactly what creation wrote.
enum FillKind {
    FILL_SEG,       // a projection segment: rows [n0, n0 + N), columns [k0, k0 + K) of the [.][ld] matrix at element `off`,
                    // repacked (qtype QT_NONE: `kb` f16 blocks per tile into rows of dst_kb blocks) or quantised
    FILL_VEC,       // `count` elements from `off` as f32 * scale + bias
    FILL_DECAY,     // `count` elements from `off` as the v5 decay table exp(-exp(x))
    FILL_FOLD,      // the k-major copy of time_decay_w2 rows n0 .. n0 + 64 N - 1 ([C][K] as stored, N heads, K = Dd)
    FILL_RAW,       // the `count` halves as stored
    FILL_INIT,      // State::init rows of layer `layer` from a time_state tensor (F16, BF16 or F32; read on the host)
};
static_assert(FILL_SEG == B200RWKV_FILL_SEG && FILL_VEC == B200RWKV_FILL_VEC && FILL_DECAY == B200RWKV_FILL_DECAY &&
                  FILL_FOLD == B200RWKV_FILL_FOLD && FILL_RAW == B200RWKV_FILL_RAW && FILL_INIT == B200RWKV_FILL_INIT,
              "b200rwkv_fill_info.kind is the FillKind");
struct Fill {
    int kind = FILL_RAW;
    size_t off = 0, count = 0;
    int ld = 0, n0 = 0, N = 0, k0 = 0, K = 0, tiles = 0, kb = 0, dst_kb = 0, qtype = QT_NONE, layer = 0;
    float scale = 1.f, bias = 0.f;
    void* dst = nullptr;
    float* scales = nullptr;        // FP8: the segment's row scales
    // what b200rwkv_debug_fill reads back beside `dst`: the plan (B200RWKV_PLAN_*) and a W' segment's adapter tail blocks,
    // `ad_tail` per tile row at `tails`, rows tails_kb blocks apart (the fills leave them alone)
    int plan = B200RWKV_PLAN_BASE, ad_tail = 0, tails_kb = 0;
    const uint8_t* tails = nullptr;
};

struct GemmLaunch {
    GemmParams p;
    int grid = 0;
    int grid_wide = 0;         // grid of steps with >= 64 tokens: whole tiles per CTA (see make_launch)
    int total_tiles = 0;
    size_t weight_bytes = 0;   // algorithmic (unpadded) weight bytes streamed (f16, or codes + block parameters)
    int qtype = QT_NONE;       // weight format of every segment of the launch (qgemm.cuh)
    // the plan's inputs, kept during build only: the adapter plans are made from them (b200rwkv_engine::ad_launch)
    std::vector<SegDesc> src;
    int force_grid = 0;
};


struct A16Buf {
    __half* p = nullptr;
    size_t halves_per_matrix = 0;
};

// What a step launches for one layer.  Decode-shaped steps (MT == 1) of a layer with a front half run it in place of LN1
// and the `lora` launches; every step then runs `pre`, WKV, O, LN2 and `ffn`.
struct Layer {
    LnMixParams ln1, ln2;
    // v6 decode front half (pre6.cuh: LN1 + token shift + ddlerp LoRA in one launch), when the model fits pre6_kernel.  Its
    // `ln` stays empty: the launch takes LN1's parameters, whose residual partials finalize_tp wires after build.
    bool has_pre6 = false;
    Pre6Params pre6{};
    std::vector<GemmLaunch> lora;   // v6 ddlerp LoRA W1, W2: after LN1 on the steps that do not run the front half
    std::vector<GemmLaunch> pre;    // launches every step runs between LN1 (or the front half) and WKV
    WkvParams wkv;
    GemmLaunch o;
    std::vector<GemmLaunch> ffn;    // launches after LN2
};

// The same layer on steps with a bound adapter: `pre`, `o` and `ffn` as in Layer, with every launch that holds an adapted
// projection replaced by its W' plan, and one shrink launch in front of each of those launches (nproj 0: none).
struct AdLayer {
    std::vector<GemmLaunch> pre;
    GemmLaunch o;
    std::vector<GemmLaunch> ffn;
    AdapterParams s_pre, s_o, s_fk, s_fv;
};

struct Profiler {
    struct Rec { int cls; Event a, b; };
    std::vector<Rec> recs;
    size_t weight_bytes = 0;        // algorithmic weight bytes of the projection launches enqueued
};

struct Snapshot { Buf<float> buf, logits; };   // CachedItem {state, output} on the device (run.rs:199-205)

// The LN-stage kernel a launch picked (b200rwkv_ln_args::kernel_out): kernel, its NV (float4 per thread of the per-token
// kernels) or Dm / 16 (pre6_kernel), and whether it wrote split (hi + lo) operands.
// LNK_MIX_CLUSTER_WIDE / LNK_PRE6_WIDE: the batch-invariant mode's variants for steps of 17..128 tokens.
enum LnKernel { LNK_EMBED = 0, LNK_MIX = 1, LNK_MIX_CLUSTER = 2, LNK_PRE6 = 3, LNK_OUT = 4, LNK_MIX_CLUSTER_WIDE = 5, LNK_PRE6_WIDE = 6 };
struct LnPick { int kernel, variant, split; };
// The launch shape of one step (b200rwkv_engine::step_shape): MT token tiles of 16 rows and MTR row tiles of the head (0: no
// output rows), `rows` = 16 * MT rows of the per-token buffers, and the token rows th / th_rows of the step's A16 operands and
// of the head's operand.  `split`: the operands hold hi + lo f16 rows (th = th_rows = 32).  `ad`: a slot of the step is bound
// to an unblended adapter, so the step runs the adapter plans and their shrink launches.  `snap`: the step holds snapshots
// (b200rwkv_infer_snapshots), so its LN stages, WKV and ln_out also write them and it ends with the snapshot rows' head
// launch over MTX row tiles (0: every snapshot token has an output row already) and their copy into the snapshots.
struct StepShape { int MT, MTR, rows, th, th_rows; bool split; bool ad = false; bool snap = false; int MTX = 0; };

// The A16 layout (common.cuh) on the host.  a16_halves: halves of one matrix of K columns.  a16_pack / a16_unpack move `ncols`
// columns of token rows between a caller's dense array and consecutive A16 matrices of K columns and `tr` token rows each (the
// last matrix may be partial): column k of matrix j, row m is dense[j * mat_ld + m * row_ld + k].  a16_pack moves all `tr`
// rows, a16_unpack the first `nrows` (any nrows <= A16_MAX_ROWS stays inside each matrix).
static inline size_t a16_halves(int K) { return (size_t)cdiv(K, GEMM_BK) * A16_KB_HALVES; }
static std::vector<uint16_t> a16_pack(const uint16_t* dense, int ncols, int K, int tr, size_t mat_ld, size_t row_ld) {
    const size_t st = a16_halves(K);
    std::vector<uint16_t> b(st * cdiv(ncols, K), 0);
    for (int c = 0; c < ncols; ++c) {
        const int j = c / K, k = c - j * K;
        for (int m = 0; m < tr; ++m) b[j * st + a16_index(m, k, tr)] = dense[j * mat_ld + m * row_ld + k];
    }
    return b;
}
static void a16_unpack(const std::vector<uint16_t>& b, int ncols, int K, int tr, int nrows, size_t mat_ld, size_t row_ld,
                       uint16_t* dense) {
    const size_t st = a16_halves(K);
    for (int c = 0; c < ncols; ++c) {
        const int j = c / K, k = c - j * K;
        for (int m = 0; m < nrows; ++m) dense[j * mat_ld + m * row_ld + k] = b[j * st + a16_index(m, k, tr)];
    }
}
// float4 per thread of the per-token LN kernels: the NV that ln_mix_row / embed_row / ln_out_row dispatch to
static inline int ln_nv(int C) {
    const int nv = (C + 4 * LN_THREADS - 1) / (4 * LN_THREADS);
    return nv <= 1 ? 1 : nv == 2 ? 2 : nv <= 4 ? 4 : 8;
}
// the cluster LN kernels hold one float4 per thread of each of the 8 channel slices
static inline bool ln_cluster_fits(int C) { return C % (4 * PRE_CLUSTER) == 0 && C / (4 * PRE_CLUSTER) <= PRE_THREADS; }
// pre6_kernel: LoRA rank Dm as its KD = Dm / 16 instantiations, 16-wide k steps in every 8-way K slice, W1 fragments in registers
static inline bool pre6_fits(int Dm, int C) { return (Dm == 32 || Dm == 64) && C % 128 == 0 && C <= PRE_MAX_C; }

}  // namespace b200

using namespace b200;

// In-process tensor parallelism (b200rwkv_create_ex with num_devices > 1): the handle the host holds is rank 0's engine; it
// owns the other ranks and one worker thread per rank.  Every SPMD entry point fans out to all ranks CONCURRENTLY (the ranks'
// kernels rendezvous with each other over NVLink, so one thread issuing rank after rank would deadlock on its first
// stream synchronisation) and returns rank 0's result: the reference's single `Runtime` object (run.rs:1230-1234).
struct Group {
    std::vector<b200rwkv_engine*> ranks;      // [world]; ranks[0] is the handle itself
    std::vector<std::thread> workers;         // ranks 1..world-1 (rank 0's share runs on the calling thread)
    std::mutex m;
    std::condition_variable cv;
    std::function<int32_t(int)> job;
    uint64_t gen = 0;
    int pending = 0;
    bool stop = false;
    std::vector<int32_t> status;
    std::vector<std::string> errs;
    std::mutex call_mu;                       // one fan-out at a time

    void start(int world);
    void shutdown();
    int32_t spmd(const std::function<int32_t(int)>& fn);
};

struct b200rwkv_engine {
    std::unique_ptr<Group> group;             // set on rank 0 of an in-process tensor-parallel engine
    b200rwkv_info info;
    int dev = 0, rank = 0, world = 1, num_sms = 132;
    int S = 0, chunk = 0, maxT = A16_MAX_ROWS, precision = 0;      // steps of up to 128 tokens
    int L = 0, C = 0, F = 0, V = 0, H = 0, N = 64, Cl = 0, Hl = 0, Fl = 0, Vl = 0;
    int split_att = 1, split_ffn = 1;
    // tensor parallel: one symmetric comm block per rank (partials, gate block, logits shard, flags)
    uint8_t* comm_base = nullptr;
    size_t comm_bytes = 0, off_part_att = 0, off_part_ffn = 0, off_rr = 0, off_logits = 0, off_flags = 0;
    uint8_t* peer_base[8] = {nullptr};
    bool peer_ipc[8] = {false};       // peer_base[q] was opened with cudaIpcOpenMemHandle (closed in the destructor)
    bool connected = false;
    TpBar tpbar;
    unsigned* d_epoch = nullptr;
    Stream stream, sm_stream;
    std::vector<Buf<void>> allocs;

    // model
    __half* emb = nullptr;
    EmbedParams embed;
    std::vector<Layer> layers;
    LnOutParams lnout;
    GemmLaunch head;
    // b200rwkv_head_format: the head's plan over quantised codes of head.weight (plan.qtype QT_NONE: none, the f16 head runs)
    // and its copy for the snapshot rows (set once snap_setup has run).  The f16 head stays resident: NONE returns to it.
    struct QHead {
        GemmLaunch plan, snap;
        Buf<uint8_t> codes;                       // code blocks, then (FP8) the row scales
        Buf<unsigned> counters, snap_counters;
    };
    QHead qhead;
    // the head launch of a step (ad: a slot of it is bound), and of its snapshot rows
    const GemmLaunch& head_plan(bool ad) const { return qhead.plan.qtype != QT_NONE ? qhead.plan : ad ? ad_head : head; }
    const GemmLaunch& snap_head_plan(bool ad) const { return qhead.plan.qtype != QT_NONE ? qhead.snap : ad ? snap_ad_head : snap_head; }
    void set_head_format(int qtype);

    // state
    float *att_shift = nullptr, *ffn_shift = nullptr, *wkv_state = nullptr, *d_api = nullptr;
    std::vector<float> init_state;     // API layout, empty => zeros
    std::map<uint64_t, Snapshot> snaps;
    uint64_t next_snap = 1;
    // b200rwkv_infer_snapshots, set up on first use (snap_setup).  One device block per snapshot step, uploaded like the
    // step metadata: [snap_meta_bytes] a copy of the step's metadata whose output rows are the snapshot tokens without one
    // (R, out_tok, tok_outrow: the rows of snap_head) | [maxT] record of each token row or null | [maxT] logits row the
    // snapshot row comes from | [maxT] the snapshot's row or null.
    size_t snap_meta_bytes = 0, snap_bytes = 0;
    Buf<uint8_t> snap_dev;
    HostBuf<uint8_t> snap_host;      // [META_RING][snap_bytes]
    A16Buf a_snap_head;
    Buf<float> snap_logits;          // [maxT][V]: rows of snap_head
    GemmLaunch snap_head, snap_ad_head;      // head / ad_head over a_snap_head into snap_logits
    AdapterParams s_snap_head;
    float* const* snap_rec_dev() const { return reinterpret_cast<float* const*>(snap_dev.p + snap_meta_bytes); }
    void snap_sizes() {
        snap_meta_bytes = (meta_ints * 4 + 15) & ~(size_t)15;
        snap_bytes = snap_meta_bytes + 3 * (size_t)maxT * sizeof(void*);
    }
    void snap_setup();
    GemmLaunch snap_rebase(const GemmLaunch& g, unsigned* counters) const;
    // one snapshot token of a step: its token row, its record, the snapshot's logits row (null: none)
    struct SnapTok { int t; float* rec; float* row; };
    int fill_snap(uint8_t* hs, const int* hm, int T, const std::vector<SnapTok>& tk) const;
    struct SnapPlan { int n; const int32_t* entry; const int32_t* tok; uint64_t* ids; };

    // activations
    float *x_a = nullptr, *x_b = nullptr, *xx1 = nullptr, *sx1 = nullptr, *xx2 = nullptr;
    float *f_r = nullptr, *f_k = nullptr, *f_v = nullptr, *f_g = nullptr, *f_w = nullptr, *f_a = nullptr, *f_nu = nullptr,
          *f_vfirst = nullptr, *f_rr = nullptr, *part_att = nullptr, *part_ffn = nullptr, *d_logits = nullptr, *d_hidden = nullptr;
    A16Buf a_x[6], a_lora[5], a_out, a_kk, a_head;
    float* gemm_ws = nullptr;
    size_t gemm_ws_floats = 0;

    // step plumbing
    static constexpr int META_RING = 4;
    Event meta_ev[META_RING];
    bool hidden_keep = false;          // b200rwkv_keep_hidden: accumulate the hidden rows of every token of an infer call
    Buf<float> d_hidden_all;
    int hidden_rows = 0;
    // b200rwkv_keep_hidden_layers: the residual stream after chosen layers for every token of an infer call.  LN1 of layer
    // l + 1 writes the rows of layer l into the step buffer d_hid_tab[l] points to (null: not recorded); layer L - 1 comes
    // from ln_out_kernel's d_hidden.  After every step the rows go to their entry's place in hid_all.
    static constexpr int HID_MAX_LAYERS = 8;
    std::vector<int> hid_layers;       // recorded layers, in the order the caller gave them
    float** d_hid_tab = nullptr;       // [L]
    float* hid_step = nullptr;         // [HID_MAX_LAYERS][maxT][C], step buffer k belongs to hid_layers[k]
    Buf<float> hid_all;                // [hid_layers.size()][tokens of the call][C]
    std::vector<int> hid_last;         // layers recorded by the most recent infer call (the layout of hid_all)
    size_t hid_last_rows = 0;
    const float* hid_step_src(int k) const { return hid_layers[k] == L - 1 ? d_hidden : hid_step + (size_t)k * maxT * C; }
    // b200rwkv_keep_hidden_pooled: one row per entry and pooled layer, reduced by hidden_pool_kernel after every step.  A
    // pooled layer's rows are recorded like a kept layer's: into the kept layer's step buffer where keep_hidden_layers asked
    // for it too, else into pool_step (so a layer only pooling asked for is never gathered token by token).
    std::vector<int> pool_layers;      // pooled layers, in the order the caller gave them
    int pool_mode = B200RWKV_POOL_LAST;
    float* pool_step = nullptr;        // [POOL_MAX_LAYERS][maxT][C], step buffer k belongs to pool_layers[k]
    float* pool_rows = nullptr;        // [POOL_MAX_LAYERS][S][C]: row (k, i) belongs to pool_layers[k] and entry i of the call
    const float* pool_src[POOL_MAX_LAYERS] = {nullptr};     // where a step's rows of pool_layers[k] are (set by upload_hid_tab)
    Buf<PoolEntry> pool_dev;           // the call's (entry, step) list, one slice per launch; grown on demand
    HostBuf<PoolEntry> pool_host;
    std::vector<int> pool_last;        // layers pooled by the most recent infer call
    std::vector<int32_t> pool_last_ntok;       // its entries' token counts
    void upload_hid_tab();
    int* d_meta = nullptr;
    HostBuf<int> h_meta;
    size_t meta_ints = 0;
    struct StepGraph { GraphExec exec; long long launches; };     // a captured step graph and the kernels it launches
    std::map<int, StepGraph> graphs;
    long long launch_total = 0;                // kernels launched by this engine's steps since creation
    long long launches_last_step = 0;
    int last_T = 0;                    // tokens of the most recent step
    StepShape last_sh{1, 0, 16, 16, 16, false};     // shape of the most recent step, replays included (debug_read)

    // softmax
    Buf<float> sm_in, sm_out;

    // sampling front half (sample.cuh): last logits row of every slot, candidate scratch, staging blobs
    float* d_keep = nullptr;                 // [S][V] (rank 0)
    std::vector<char> keep_valid;            // slot has a logits row (guarded by keep_mu)
    std::mutex keep_mu;
    Event step_done;                         // recorded on `stream` after every step: the sampling stream waits on it
    float* tk_cand_x = nullptr; unsigned* tk_cand_id = nullptr; float2* tk_stats = nullptr;
    unsigned* tk_out_id = nullptr; float* tk_out_p = nullptr;
    Buf<uint8_t> tk_dev;
    HostBuf<uint8_t> tk_host;
    // b200rwkv_sample_probs: [nrows][V rounded up to 4] f32 rows | [nrows][segments] float2 statistics; grown on demand
    Buf<uint8_t> sp_dev;
    // scoring (b200rwkv_infer_ex, OPTION_SCORE): [ScoreRow x n | score f32 x n | argmax u32 x n], pinned host and device,
    // n = the call's scored tokens; grown on demand
    Buf<uint8_t> sc_dev;
    HostBuf<uint8_t> sc_host;
    // b200rwkv_score_top: with top_n > 0 both score buffers go on with [ids u32 x n x top_n | logprobs f32 x n x top_n], and
    // every score launch is followed by the two score_top launches over the same rows, whose candidate lists go to
    // top_cand_x / top_cand_id ([max(S, maxT)][segments][128]: a launch lists at most one row per SCORE entry or per token
    // of a step).  top_last_n / top_last_rows: the setting and the scored tokens of the most recent infer call, whose lists
    // sit in sc_host.
    int top_n = 0;
    float* top_cand_x = nullptr; unsigned* top_cand_id = nullptr;
    int top_last_n = 0;
    size_t top_last_rows = 0;
    void enqueue_keep(cudaStream_t s, int MTR);
    void enqueue_snap_rows(cudaStream_t s, const StepShape& sh);
    void check_sample_slots(int nrows, const int32_t* slots, const char* who);
    SampleAdjust stage_sample_args(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok,
                                   const float* pen_val, const uint32_t* allow_bits, const int32_t* bias_off,
                                   const uint32_t* bias_tok, const float* bias_val);
    void sample_topk(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok, const float* pen_val,
                     const uint32_t* allow_bits, const int32_t* bias_off, const uint32_t* bias_tok, const float* bias_val,
                     int top_k, uint32_t* ids_out, float* probs_out);
    void sample_probs(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok, const float* pen_val,
                      const uint32_t* allow_bits, const int32_t* bias_off, const uint32_t* bias_tok, const float* bias_val,
                      float* probs_out);

    std::mutex mu, sm_mu;

    // LoRA files blended into the projection weights while they are uploaded (borrowed during build only)
    struct LoraSrc { const StFile* st; float alpha; };
    std::vector<LoraSrc> loras;
    // unblended adapters (b200rwkv_create_adapters, b200rwkv_create_adapter_places): files borrowed during build only, plans
    // and A matrices kept.  n_adapters places, ids 1..n; `ad_targets`: the kinds of matrix a places engine plans (0: the
    // matrices the files pair)
    std::vector<LoraSrc> adapters;
    int n_adapters = 0;
    uint32_t ad_targets = 0;
    std::vector<AdLayer> ad_layers;
    GemmLaunch ad_head;
    AdapterParams s_head;
    int* d_slot_adapter = nullptr;           // [S] adapter bound to each slot, 0 = the base model
    std::vector<int> slot_adapter;           // host copy (the infer task's)
    // What b200rwkv_load_adapter / unload_adapter write, per matrix with a W' plan: its W' segment (`tiles` rows of KB weight
    // blocks; place b's tail block is block kbw + b - 1 of each row), its entry `proj` of the shrink launch `sp`, and each
    // place's A rows ([128][K] f16, reserved at creation)
    struct AdMatrix {
        std::string name;                    // "blocks.<l>.<kind>" or "head"
        int N, K;
        uint8_t* W;
        int tiles, KB, kbw;
        AdapterParams* sp;
        int proj;
        __half* A[AD_MAX];
    };
    std::vector<AdMatrix> ad_mats;
    std::vector<char> place_full;            // [n_adapters]: the place holds an adapter (bind_adapter refuses an empty one)
    std::map<std::string, StTensor> model_shapes;     // the model's tensor names and shapes, for load_adapter's file checks
    uint8_t* ad_stage = nullptr;             // load_adapter's staging: [N][128] f16 tail columns | their repacked blocks
    size_t ad_stage_cols = 0;                // bytes of the first part
    void set_place_rank(const AdMatrix& m, int id, int r);
    void load_place(int id, const StFile& f, float alpha);
    void unload_place(int id);
    void drop_adapter_graphs();
    bool step_bound(const std::vector<int>& slots) const {
        for (int s : slots)
            if (n_adapters && s >= 0 && s < S && slot_adapter[s]) return true;
        return false;
    }
    GemmLaunch ad_launch(const GemmLaunch& base, AdapterParams& sp);
    void enqueue_shrink(const AdapterParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof);
    void check_loras(const StFile& model) const;
    void blend_loras(const StTensor& t);
    bool had_loras = false;                  // LoRA files were blended at creation (a weight update cannot redo the blend)

    // Every weight fill of the build, by the tensor it reads (FillKind), and the f16 staging buffer they read from: held
    // during the build and during a weight update only, sized to the largest tensor of the call
    std::map<std::string, std::vector<Fill>> fills;
    Buf<__half> d_tmp;
    // one tensor of a fill_weights call: host bytes (an image), or dense device bytes in a B200RWKV_DTYPE_*
    struct WeightIn { std::string name; const StTensor* host; const void* dev; int dtype; int64_t numel; };
    void fill_weights(const std::vector<WeightIn>& in);
    void run_fill(const Fill& f, const __half* src, cudaStream_t s);
    void put_adapter_tails(const SegDesc& d, int ke, uint8_t* dst, int dst_kb);

    ~b200rwkv_engine();
    void* dalloc(size_t bytes, bool zero = true);
    void build(const StFile& st);
    float* vec_f32(const StFile& st, const std::string& name, size_t off, size_t count, float scale = 1.f, float bias = 0.f);
    A16Buf a16_alloc(int K, int nmat = 1);
    GemmLaunch make_launch(std::vector<SegDesc>& segs, int force_grid = 0, int qtype = QT_NONE, int plan = B200RWKV_PLAN_BASE);
    int quant_layers = 0, quant_type = QT_NONE;     // the first `quant_layers` layers hold Int8 / NF4 / FP8 / Int4 projection matrices
    // b200rwkv_options.quant_adapters: adapters may pair matrices of the quantised layers (quantised W' plans: the base plan's
    // code blocks and f16 tail blocks, GemmParams::tails)
    bool quant_adapters = false;
    // quant_layers as the adapter checks see it: no layer refuses adapters with quant_adapters
    int ad_quant_layers() const { return quant_adapters ? 0 : quant_layers; }
    int pick_split(int K, int tiles) const;
    void finalize_tp();
    template <typename P, typename... X>
    void launch_k(void (*kern)(P, X...), dim3 grid, dim3 block, size_t smem, const P& params, int cls, cudaStream_t s, Profiler* prof,
                  X... extra);
    bool split_on = false;        // precision 1: split (hi + lo f16) projection operands, every step decode-shaped
    bool split_act = false;
    bool ln_cluster_ok = false;   // the decode-shaped cluster LN kernels of pre6.cuh fit the model
    // b200rwkv_options.batch_invariant: steps of more than 16 tokens compute every token with the decode step's arithmetic
    // (DESIGN.md §6, batch-invariant engines): the cluster LN stages and the RWKV-6 front half in their WIDE variants, every
    // projection on its `grid` plan (the K split of a decode step)
    bool batch_inv = false;
    unsigned* pre_gbar = nullptr;
    int launch_cluster = 0;                       // consumed by the next launch_k
    // profiling aid (b200rwkv_profile_insitu): 8 globaltimer stamps of CTA 0 per launch of the per-op chain
    unsigned long long* d_step_trace = nullptr;
    std::vector<int> step_trace_types;
    static constexpr int STEP_TRACE_MAX = 1024;
    static constexpr int STEP_TRACE_ROW = 512;     // 8 stamps of CTA 0 + {SM id, last MMA, exit} of every projection CTA
    bool trace_capture = false;                    // stamps are wired into the launches being enqueued / captured right now
    std::vector<long long> step_trace_bytes;       // algorithmic weight bytes of each traced projection launch
    unsigned long long* tr_next(int label) {
        if (!d_step_trace || !trace_capture || launches_last_step >= STEP_TRACE_MAX) return nullptr;
        if ((int)step_trace_types.size() <= launches_last_step) step_trace_types.resize(launches_last_step + 1);
        step_trace_types[launches_last_step] = label;
        return d_step_trace + (size_t)STEP_TRACE_ROW * launches_last_step;
    }
    StepShape step_shape(int T, int R) const;
    // `head`: the head projection, over the step's output rows
    void launch_gemm(const GemmLaunch& g, const StepShape& sh, cudaStream_t s, Profiler* prof, bool head = false);
    void launch_wkv(const WkvParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof);
    // LN stages of a step; each returns which kernel it launched
    LnPick launch_embed(const EmbedParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof);
    LnPick launch_ln(const LnMixParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof);
    LnPick launch_pre6(const Pre6Params& q, const StepShape& sh, cudaStream_t s, Profiler* prof);
    LnPick launch_ln_out(const LnOutParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof);
    void enqueue_step(cudaStream_t s, const StepShape& sh, Profiler* prof);
    void run_step(const StepShape& sh);
    int fill_meta(int* m, const std::vector<int>& slots, const std::vector<int>& counts, const std::vector<const uint32_t*>& toks,
                  const std::vector<int>& outmode /*0 none,1 last,2 full*/, int* R_out);
    // score == nullptr: b200rwkv_infer, which refuses OPTION_SCORE
    struct ScoreOut { float* score; uint32_t* argmax; };
    // snap: b200rwkv_infer_snapshots (null or n == 0: none)
    void infer(int nslot, const int32_t* slot, const int32_t* ntok, const uint32_t* tokens, const int32_t* option,
               float* logits_out, size_t cap, int32_t* rows_out, const ScoreOut* score = nullptr, const SnapPlan* snap = nullptr);
    void state_xform(int slot, bool import, float* snap = nullptr);
};

// The members release their resources after this body, once the device has finished every queued use of them.
b200rwkv_engine::~b200rwkv_engine() {
    cudaSetDevice(dev);
    cudaDeviceSynchronize();
    for (int q = 0; q < 8; ++q)
        if (peer_ipc[q] && peer_base[q]) cudaIpcCloseMemHandle(peer_base[q]);
}

void* b200rwkv_engine::dalloc(size_t bytes, bool zero) {
    bytes = std::max<size_t>(bytes, 16);
    allocs.emplace_back(bytes);
    if (zero) CK(cudaMemset(allocs.back(), 0, bytes));
    return allocs.back();
}

static bool ends_with(const std::string& s, const std::string& suf) {
    return s.size() >= suf.size() && s.compare(s.size() - suf.size(), suf.size(), suf) == 0;
}

// The projection kinds a LoRA pair may address; bit i of a B200RWKV_TARGET_* mask is kind i, B200RWKV_TARGET_HEAD the head.
static const char* const LORA_KINDS[] = {".att.receptance", ".att.key", ".att.value", ".att.gate", ".att.output", ".ffn.key",
                                         ".ffn.value", ".ffn.receptance"};
static const uint32_t AD_TARGET_ALL = (1u << 9) - 1;
static uint32_t ad_target_bit(const std::string& base) {
    if (base == "head") return B200RWKV_TARGET_HEAD;
    for (int i = 0; i < 8; ++i)
        if (ends_with(base, LORA_KINDS[i])) return 1u << i;
    return 0;
}
// the matrix `base` sits in one of the first `quant_layers` layers, which hold quantised projection matrices
static bool in_quant_layer(const std::string& base, int quant_layers, int quant_type) {
    const int layer = base.compare(0, 7, "blocks.") == 0 ? atoi(base.c_str() + 7) : -1;
    return quant_type != QT_NONE && layer >= 0 && layer < quant_layers;
}
// Matrices an engine from b200rwkv_create_adapter_places plans a W' for: every 2-D `<base>.weight` of the model of a targeted
// kind outside the first `quant_layers` layers (0 with quant_adapters).
static std::vector<std::string> ad_place_matrices(const std::map<std::string, StTensor>& model, uint32_t targets,
                                                  int quant_layers, int quant_type) {
    std::vector<std::string> out;
    for (auto& kv : model) {
        if (!ends_with(kv.first, ".weight") || kv.second.shape.size() != 2) continue;
        const std::string base = kv.first.substr(0, kv.first.size() - 7);
        if ((ad_target_bit(base) & targets) && !in_quant_layer(base, quant_layers, quant_type)) out.push_back(base);
    }
    return out;
}
static const StTensor* st_find(const std::map<std::string, StTensor>& m, const std::string& name) {
    auto it = m.find(name);
    return it == m.end() ? nullptr : &it->second;
}

// Every `<base>.lora.0/.lora.1` pair of a LoRA file must address a projection matrix this engine blends (the matrices that
// blend_loras changes as fill_weights reads them); anything else is refused loudly rather than ignored.  `model`: the model's
// tensors (names and shapes are what is read).
static void check_lora_files(const std::map<std::string, StTensor>& model, const std::vector<b200rwkv_engine::LoraSrc>& files) {
    for (const b200rwkv_engine::LoraSrc& lo : files) {
        int pairs = 0;
        for (auto& kv : lo.st->tensors) {
            const std::string& n = kv.first;
            if (ends_with(n, ".lora.1")) continue;
            if (!ends_with(n, ".lora.0")) {
                REQUIRE(!st_find(model, n), B200RWKV_ERR_UNSUPPORTED, "LoRA file carries a full tensor (" + n + "): only low-rank pairs on projection matrices are blended");
                continue;
            }
            const std::string base = n.substr(0, n.size() - 7);
            const bool good = ad_target_bit(base) != 0;
            REQUIRE(good && st_find(model, base + ".weight"), B200RWKV_ERR_UNSUPPORTED, "LoRA on " + base + " is not supported (projection matrices only)");
            REQUIRE(lo.st->find(base + ".lora.1"), B200RWKV_ERR_INVALID, "LoRA file: " + base + ".lora.1 is missing");
            ++pairs;
        }
        REQUIRE(pairs > 0, B200RWKV_ERR_INVALID, "LoRA file holds no <name>.lora.0 / <name>.lora.1 pairs");
    }
}
void b200rwkv_engine::check_loras(const StFile& model) const { check_lora_files(model.tensors, loras); }

// Adapter files (b200rwkv_create_adapters, b200rwkv_load_adapter), host only: the load-time blend's refusals, then every
// pair's halves, dtypes and shapes against the model, the rank (one 128-wide k block of W'), and no pair on a matrix of one
// of the first `quant_layers` layers (0 with quant_adapters: every layer takes adapters).
static void check_adapter_files(const std::map<std::string, StTensor>& model, const std::vector<b200rwkv_engine::LoraSrc>& files,
                                int quant_layers, int quant_type) {
    check_lora_files(model, files);
    for (const b200rwkv_engine::LoraSrc& lo : files)
        for (auto& kv : lo.st->tensors) {
            const std::string& n = kv.first;
            if (!ends_with(n, ".lora.0") && !ends_with(n, ".lora.1")) continue;
            const std::string base = n.substr(0, n.size() - 7);
            const StTensor* a = lo.st->find(base + ".lora.0");
            const StTensor* b = lo.st->find(base + ".lora.1");
            REQUIRE(a && b, B200RWKV_ERR_INVALID, "adapter file: " + base + " has only one of .lora.0 / .lora.1");
            if (n != base + ".lora.0") continue;
            const StTensor* w = st_find(model, base + ".weight");
            REQUIRE(w && w->shape.size() == 2, B200RWKV_ERR_UNSUPPORTED, "adapter on " + base + " is not supported (projection matrices only)");
            REQUIRE(a->dtype == "F16" && b->dtype == "F16", B200RWKV_ERR_UNSUPPORTED, "adapter tensors must be F16: " + base);
            REQUIRE(a->shape.size() == 2 && b->shape.size() == 2 && b->shape[0] == w->shape[0] && a->shape[0] == w->shape[1] &&
                        a->shape[1] == b->shape[1] && a->shape[1] >= 1,
                    B200RWKV_ERR_INVALID, "adapter shapes do not match " + base + ".weight (expected lora.0 [in, r], lora.1 [out, r])");
            REQUIRE(a->shape[1] <= AD_MAX_RANK, B200RWKV_ERR_UNSUPPORTED,
                    "adapter rank " + std::to_string(a->shape[1]) + " on " + base + " is above 128");
            REQUIRE(a->shape[0] % 8 == 0, B200RWKV_ERR_UNSUPPORTED, "adapter on " + base + ": input width must be a multiple of 8");
            REQUIRE(!in_quant_layer(base, quant_layers, quant_type), B200RWKV_ERR_UNSUPPORTED,
                    "adapter on " + base + ": its layer is quantised (adapters need f16 projection matrices)");
        }
}

// The load-time weight kernels with the launch shapes the build gives them; b200rwkv_op_weight runs these same launches.
static void launch_lora_blend(int num_sms, __half* W, const __half* B, const __half* At, int out, int in, int r, float alpha) {
    lora_blend_kernel<<<num_sms * 8, 256>>>(W, B, At, out, in, r, alpha);
    CK(cudaGetLastError());
}
static void launch_f16_to_f32(const __half* src, float* dst, size_t count, float scale, float bias, cudaStream_t s = 0) {
    f16_to_f32_kernel<<<cdiv((int)count, 256), 256, 0, s>>>(src, dst, count, scale, bias);
    CK(cudaGetLastError());
}
static void launch_decay_table(const __half* src, float* dst, int n, cudaStream_t s = 0) {
    decay_table_kernel<<<cdiv(n, 256), 256, 0, s>>>(src, dst, n);
    CK(cudaGetLastError());
}
// rows [n0, n0 + N) and columns [k0, k0 + K) of src [.][ld] into ceil(N / 128) x ceil(K / 128) stage blocks at dst, dst_kb
// blocks per tile row (0: ceil(K / 128))
static void launch_repack(int num_sms, const __half* src, int ld, int n0, int k0, int N, int K, uint4* dst,
                          cudaStream_t s = 0, int dst_kb = 0) {
    const int tiles = cdiv(N, GEMM_BN), KB = cdiv(K, GEMM_BK);
    const size_t nchunk = (size_t)tiles * KB * (GEMM_WBYTES / 16);
    const int grid = (int)std::min<size_t>((nchunk + 255) / 256, (size_t)num_sms * 16);
    repack_weight_kernel<<<grid, 256, 0, s>>>(src, ld, n0, k0, N, K, tiles, KB, dst_kb > 0 ? dst_kb : KB, dst);
    CK(cudaGetLastError());
}

void b200rwkv_engine::blend_loras(const StTensor& t) {
    if (loras.empty() || !ends_with(t.name, ".weight") || t.shape.size() != 2) return;
    const std::string base = t.name.substr(0, t.name.size() - 7);
    const int out = (int)t.shape[0], in = (int)t.shape[1];
    for (const LoraSrc& lo : loras) {
        const StTensor* a = lo.st->find(base + ".lora.0");
        const StTensor* b = lo.st->find(base + ".lora.1");
        if (!a || !b) continue;
        REQUIRE(a->dtype == "F16" && b->dtype == "F16", B200RWKV_ERR_UNSUPPORTED, "LoRA tensors must be F16: " + base);
        REQUIRE(a->shape.size() == 2 && b->shape.size() == 2 && b->shape[0] == out && a->shape[0] == in && a->shape[1] == b->shape[1] &&
                    a->shape[1] >= 1 && a->shape[1] <= 4096,
                B200RWKV_ERR_INVALID, "LoRA shapes do not match " + t.name + " (expected lora.0 [in, r], lora.1 [out, r])");
        const int r = (int)a->shape[1];
        Buf<__half> da(a->nbytes), db(b->nbytes);
        CK(cudaMemcpy(da, a->data, a->nbytes, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(db, b->data, b->nbytes, cudaMemcpyHostToDevice));
        launch_lora_blend(num_sms, d_tmp, db, da, out, in, r, lo.alpha);
        CK(cudaDeviceSynchronize());
    }
}

// an f32 vector, filled by fill_weights
float* b200rwkv_engine::vec_f32(const StFile& st, const std::string& name, size_t off, size_t count, float scale, float bias) {
    const StTensor& t = st.get(name);
    REQUIRE((size_t)t.numel() >= off + count, B200RWKV_ERR_INVALID, "tensor too small: " + name);
    Fill f;
    f.kind = FILL_VEC; f.off = off; f.count = count; f.scale = scale; f.bias = bias;
    f.dst = dalloc(count * 4, false);
    fills[name].push_back(f);
    return (float*)f.dst;
}

A16Buf b200rwkv_engine::a16_alloc(int K, int nmat) {
    A16Buf b;
    b.halves_per_matrix = a16_halves(K);     // whole 128-wide k blocks, zero padded
    b.p = (__half*)dalloc(b.halves_per_matrix * 2 * nmat, true);
    return b;
}

// The adapter tail blocks of a W' segment: E [N][ke] holds f16(alpha * lora.1) of every adapter file with a pair on the
// segment's matrix in columns 128 a .. (zeros past the rank, and for an adapter without a pair here: adapter places are
// created empty), re-tiled into rows of dst_kb blocks at dst.  The weight fills leave these blocks alone.
void b200rwkv_engine::put_adapter_tails(const SegDesc& d, int ke, uint8_t* dst, int dst_kb) {
    const std::string base = d.t->name.substr(0, d.t->name.size() - 7);
    Buf<__half> E((size_t)d.N * ke * 2);
    CK(cudaMemset(E, 0, E.bytes));
    for (int a = 0; a < (int)adapters.size(); ++a) {
        const StTensor* b = adapters[a].st->find(base + ".lora.1");
        if (!b) continue;
        const int r = (int)b->shape[1];
        std::vector<__half> h((size_t)d.N * r);
        memcpy(h.data(), b->data + (size_t)d.n0 * r * 2, h.size() * 2);
        for (__half& v : h) v = __float2half_rn(adapters[a].alpha * __half2float(v));
        CK(cudaMemcpy2D(E + (size_t)a * GEMM_BK, (size_t)ke * 2, h.data(), (size_t)r * 2, (size_t)r * 2, d.N, cudaMemcpyHostToDevice));
    }
    launch_repack(num_sms, E, ke, 0, 0, d.N, ke, reinterpret_cast<uint4*>(dst), 0, dst_kb);
    CK(cudaDeviceSynchronize());
}

// Algorithmic bytes of an [N][K] matrix in a quantised format: codes + block parameters (FP8: one f32 scale per row)
static size_t quant_matrix_bytes(int qtype, size_t N, size_t K) {
    if (qtype == QT_FP8) return N * K + N * 4;
    if (qtype == QT_INT4) return N * K / 2 + N * (K / 128) * 4;
    return qtype == QT_INT8 ? N * K + N * (K / 128) * 4 : N * K / 2 + N * (K / 64) * 2;
}

// The plan of one projection launch over `segs`; its weight blocks are written by the FILL_SEG fills it records.
GemmLaunch b200rwkv_engine::make_launch(std::vector<SegDesc>& segs, int force_grid, int qtype, int plan) {
    REQUIRE(!segs.empty() && (int)segs.size() <= GEMM_MAX_SEG, B200RWKV_ERR_INVALID, "internal: bad segment count");
    GemmLaunch g;
    memset(&g.p, 0, sizeof(g.p));
    g.qtype = qtype;
    const size_t blk_bytes = (size_t)q_block_bytes(qtype);
    int blk = 0, tile = 0, kbmax = 0;
    int qblk = 0, tblk = 0;        // quantised plans: code blocks and f16 tail blocks so far (GemmParams::tails)
    for (size_t i = 0; i < segs.size(); ++i) {
        SegDesc& d = segs[i];
        GemmSeg& sg = g.p.seg[i];
        sg = d.proto;
        // A16 outputs are written as whole 16-byte chunks of 8 rows (gemm.cuh epilogue)
        REQUIRE(sg.out_mode == OUT_F32 || (d.N % 8 == 0 && sg.grp % 8 == 0), B200RWKV_ERR_UNSUPPORTED,
                "LoRA ranks / hidden size must be multiples of 8");
        sg.KB = cdiv(d.K, GEMM_BK) + d.ad_tail;
        sg.tiles = cdiv(d.N, GEMM_BN);
        sg.N = d.N;
        sg.blk_begin = blk;
        sg.tile_begin = tile;
        blk += sg.tiles * sg.KB;
        tile += sg.tiles;
        kbmax = std::max(kbmax, sg.KB);
        g.p.kbq[i] = sg.KB - d.ad_tail;
        g.p.qblk[i] = qblk;
        g.p.tblk[i] = tblk;
        qblk += sg.tiles * g.p.kbq[i];
        tblk += sg.tiles * d.ad_tail;
        if (qtype == QT_NONE) g.weight_bytes += (size_t)d.N * (d.K + (size_t)d.ad_tail * GEMM_BK) * 2;
        else {
            g.weight_bytes += (size_t)d.N * d.ad_tail * GEMM_BK * 2;
            // quantisation blocks are runs of 128 (Int8, Int4) / 64 (NF4) consecutive inputs of one output row of the FULL matrix
            REQUIRE(d.K % GEMM_BK == 0 && d.k0 % GEMM_BK == 0, B200RWKV_ERR_UNSUPPORTED,
                    "quantised projections need input dimensions that are multiples of 128");
            g.weight_bytes += quant_matrix_bytes(qtype, d.N, d.K);
        }
    }
    g.p.nseg = (int)segs.size();
    g.src = segs;
    g.force_grid = force_grid;
    g.p.total_blocks = blk;
    g.total_tiles = tile;
    // FP8: the launch's row scales follow its code blocks, FP8_SCALE_BYTES per tile (fp8gemm.cuh).  A quantised plan with
    // adapter tails keeps them apart from its code blocks (GemmParams::tails); an f16 plan holds them among its blocks.
    const int wblk = qtype == QT_NONE ? blk : qblk;
    uint8_t* W = (uint8_t*)dalloc((size_t)wblk * blk_bytes + (qtype == QT_FP8 ? (size_t)tile * FP8_SCALE_BYTES : 0), false);
    g.p.W = W;
    if (qtype == QT_FP8) g.p.scales = reinterpret_cast<const float*>(W + (size_t)wblk * blk_bytes);
    if (qtype != QT_NONE && tblk) g.p.tails = (const uint8_t*)dalloc((size_t)tblk * GEMM_WBYTES, false);
    for (size_t i = 0; i < segs.size(); ++i) {
        const SegDesc& d = segs[i];
        const GemmSeg& sg = g.p.seg[i];
        const StTensor& t = *d.t;
        Fill f;
        f.kind = FILL_SEG; f.n0 = d.n0; f.N = d.N; f.k0 = d.k0; f.K = d.K; f.tiles = sg.tiles; f.kb = g.p.kbq[i]; f.qtype = qtype;
        f.plan = plan; f.ad_tail = d.ad_tail;
        if (d.slice >= 0) {
            REQUIRE(t.shape.size() == 3, B200RWKV_ERR_INVALID, "internal: slice of non-3D tensor");
            f.ld = (int)t.shape[2];
            f.off = (size_t)d.slice * t.shape[1] * t.shape[2];
            REQUIRE(d.slice < t.shape[0] && d.n0 + d.N <= t.shape[1] && d.k0 + d.K <= t.shape[2], B200RWKV_ERR_INVALID, "weight shape mismatch");
        } else {
            REQUIRE(t.shape.size() == 2, B200RWKV_ERR_INVALID, "internal: expected 2-D weight");
            f.ld = (int)t.shape[1];
            REQUIRE(d.n0 + d.N <= t.shape[0] && d.k0 + d.K <= t.shape[1], B200RWKV_ERR_INVALID, "weight shape mismatch");
        }
        if (qtype == QT_NONE) {
            // an f16 W' plan's rows are the segment's own k blocks, then its adapter tail blocks
            f.dst = W + (size_t)sg.blk_begin * GEMM_WBYTES;
            f.dst_kb = sg.KB;
            f.tails = W + (size_t)(sg.blk_begin + f.kb) * GEMM_WBYTES;
            f.tails_kb = sg.KB;
            if (d.ad_tail) put_adapter_tails(d, d.ad_tail * GEMM_BK, W + (size_t)(sg.blk_begin + f.kb) * GEMM_WBYTES, sg.KB);
        } else {
            f.dst = W + (size_t)g.p.qblk[i] * blk_bytes;
            if (qtype == QT_FP8) f.scales = const_cast<float*>(g.p.scales) + (size_t)sg.tile_begin * GEMM_BN;
            // the tail blocks alone, [tile][ad_tail], re-tiled as the f16 plan's
            f.tails = g.p.tails + (size_t)g.p.tblk[i] * GEMM_WBYTES;
            f.tails_kb = d.ad_tail;
            if (d.ad_tail) put_adapter_tails(d, d.ad_tail * GEMM_BK, const_cast<uint8_t*>(g.p.tails) + (size_t)g.p.tblk[i] * GEMM_WBYTES, d.ad_tail);
        }
        fills[t.name].push_back(f);
    }
    g.grid = std::max(1, std::min(num_sms, std::max(tile, cdiv(blk, 4))));
    g.grid = std::min(g.grid, blk);
    if (force_grid > 0) g.grid = std::min(force_grid, blk);
    else {
        // Whole tiles per CTA whenever that keeps >= 3/4 of the SMs streaming: no cross-CTA fix-up in the tail, and a grid
        // that leaves some SMs idle need not finish later than a full one, whose CTAs skew across GPCs of unequal SM counts.
        if (tile <= num_sms && tile * 4 >= num_sms * 3) g.grid = tile;
        else if (tile > num_sms)
            for (int cand = num_sms; cand * 4 >= num_sms * 3; --cand)
                if (tile % cand == 0) { g.grid = cand; break; }
    }
    // Steps of 64 / 128 tokens: a partial accumulator tile is 32 / 64 KB per contributor, and the last arriver of a cut tile
    // spends tens of microseconds summing them.  Those steps run whole tiles per CTA, even if that leaves SMs idle.
    g.grid_wide = g.grid;
    if (force_grid <= 0) {
        if (tile <= num_sms) g.grid_wide = tile;
        else
            for (int cand = num_sms; cand * 2 >= num_sms; --cand)        // several whole tiles per CTA; else keep stream-K
                if (tile % cand == 0) { g.grid_wide = cand; break; }
    }
    const int per_cta = std::max(1, blk / g.grid);
    g.p.max_contrib = cdiv(kbmax, per_cta) + 1;
    g.p.counters = (unsigned*)dalloc((size_t)tile * 4, true);
    g.p.nrows = d_meta;   // T by default
    g.p.w_lbo = GEMM_W_LBO; g.p.w_sbo = GEMM_W_SBO; g.p.a_lbo = GEMM_A_LBO; g.p.a_sbo = GEMM_A_SBO;
    gemm_ws_floats = std::max(gemm_ws_floats, (size_t)tile * g.p.max_contrib * (size_t)maxT * GEMM_BN);
    return g;
}

template <typename P, typename... X>
void b200rwkv_engine::launch_k(void (*kern)(P, X...), dim3 grid, dim3 block, size_t smem, const P& params, int cls, cudaStream_t s,
                               Profiler* prof, X... extra) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (launch_cluster > 0) {
        at[na].id = cudaLaunchAttributeClusterDimension;
        at[na].val.clusterDim.x = (unsigned)launch_cluster;
        at[na].val.clusterDim.y = 1;
        at[na].val.clusterDim.z = 1;
        ++na;
        launch_cluster = 0;
    }
    if (!prof) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = at;
    cfg.numAttrs = na;
    Event ea, eb;
    if (prof) {
        ea = new_event();
        eb = new_event();
        CK(cudaEventRecord(ea, s));
    }
    CK(cudaLaunchKernelEx(&cfg, kern, params, extra...));
    if (prof) {
        CK(cudaEventRecord(eb, s));
        prof->recs.push_back({cls, std::move(ea), std::move(eb)});
    }
    ++launches_last_step;
}

void b200rwkv_engine::launch_gemm(const GemmLaunch& g, const StepShape& sh, cudaStream_t s, Profiler* prof, bool head) {
    const int MT = head ? sh.MTR : sh.MT;
    GemmParams p = g.p;
    for (int i = 0; i < p.nseg; ++i)
        if (p.seg[i].out_mode != OUT_F32) p.seg[i].ldo = sh.th;     // A16 outputs feed a projection of this step
    if (g.qtype != QT_NONE) {
        REQUIRE(!sh.split, B200RWKV_ERR_UNSUPPORTED, "internal: quantised projections run with f16 activations");
        const int grid = MT >= 4 && !batch_inv ? g.grid_wide : g.grid;
        // W' plans (adapter tails) run the tail instantiations
        const bool tails = p.tails != nullptr;
#define FLAUNCH(MT_)                                                                                                                \
    (tails ? launch_k(fp8gemm_tail_kernel<MT_>, dim3(grid), dim3(GEMM_THREADS), Fp8GemmCfg<MT_, true>::SMEM_BYTES, p, KC_GEMM, s, prof) \
           : launch_k(fp8gemm_kernel<MT_>, dim3(grid), dim3(GEMM_THREADS), Fp8GemmCfg<MT_>::SMEM_BYTES, p, KC_GEMM, s, prof))
        if (g.qtype == QT_FP8) {
            switch (MT) { case 1: FLAUNCH(1); break; case 2: FLAUNCH(2); break; case 4: FLAUNCH(4); break; default: FLAUNCH(8); break; }
            return;
        }
#undef FLAUNCH
#define ILAUNCH(MT_)                                                                                                                  \
    (tails ? launch_k(int4gemm_tail_kernel<MT_>, dim3(grid), dim3(GEMM_THREADS), Int4GemmCfg<MT_, true>::SMEM_BYTES, p, KC_GEMM, s, prof) \
           : launch_k(int4gemm_kernel<MT_>, dim3(grid), dim3(GEMM_THREADS), Int4GemmCfg<MT_>::SMEM_BYTES, p, KC_GEMM, s, prof))
        if (g.qtype == QT_INT4) {
            switch (MT) { case 1: ILAUNCH(1); break; case 2: ILAUNCH(2); break; case 4: ILAUNCH(4); break; default: ILAUNCH(8); break; }
            return;
        }
#undef ILAUNCH
#define QLAUNCH(MT_, QT_)                                                                                                                  \
    (tails ? launch_k(qgemm_tail_kernel<MT_, QT_>, dim3(grid), dim3(QGEMM_THREADS), QGemmCfg<MT_, QT_>::SMEM_BYTES, p, KC_GEMM, s, prof) \
           : launch_k(qgemm_kernel<MT_, QT_>, dim3(grid), dim3(QGEMM_THREADS), QGemmCfg<MT_, QT_>::SMEM_BYTES, p, KC_GEMM, s, prof))
        if (g.qtype == QT_INT8) {
            switch (MT) { case 1: QLAUNCH(1, QT_INT8); break; case 2: QLAUNCH(2, QT_INT8); break; case 4: QLAUNCH(4, QT_INT8); break; default: QLAUNCH(8, QT_INT8); break; }
        } else {
            switch (MT) { case 1: QLAUNCH(1, QT_NF4); break; case 2: QLAUNCH(2, QT_NF4); break; case 4: QLAUNCH(4, QT_NF4); break; default: QLAUNCH(8, QT_NF4); break; }
        }
#undef QLAUNCH
        return;
    }
    // RING 2 = one stage less than fits, so the small kernels around a projection can share its SMs (findings r1 §7)
    const int gw = batch_inv ? g.grid : g.grid_wide;
    switch (MT) {
        case 1:
            if (sh.split) launch_k(gemm_kernel<2, 2, true>, dim3(g.grid), dim3(GEMM_THREADS), GemmCfg<2, 2>::SMEM_BYTES, p, KC_GEMM, s, prof);
            else launch_k(gemm_kernel<1, 2>, dim3(g.grid), dim3(GEMM_THREADS), GemmCfg<1, 2>::SMEM_BYTES, p, KC_GEMM, s, prof);
            break;
        case 2: launch_k(gemm_kernel<2>, dim3(g.grid), dim3(GEMM_THREADS), GemmCfg<2>::SMEM_BYTES, p, KC_GEMM, s, prof); break;
        case 4: launch_k(gemm_kernel<4>, dim3(gw), dim3(GEMM_THREADS), GemmCfg<4>::SMEM_BYTES, p, KC_GEMM, s, prof); break;
        default: launch_k(gemm_kernel<8>, dim3(gw), dim3(GEMM_THREADS), GemmCfg<8>::SMEM_BYTES, p, KC_GEMM, s, prof); break;
    }
}

// The WKV launch of one step: one CTA per (head, step entry) over min(S, rows) entries (a step has at most one entry per token;
// CTAs past the step's entries exit), decay rows and staged rows sized by the step shape, since a slot cannot hold more tokens
// than the step.  Split steps write hi + lo output rows.
void b200rwkv_engine::launch_wkv(const WkvParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    WkvParams wp = p;
    wp.kq_tile = sh.th; wp.d1_kq = sh.th;
    const int rows = sh.rows;
    const dim3 grid(wp.H, std::min(S, rows));
    const size_t sm_b = wkv_smem_bytes(wp.version, wp.version == 6 && wp.wd2t, wp.Dd, rows, sh.split);
    auto go = [&](auto kern) { launch_k(kern, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); };
    if (sh.snap) {
        switch (wp.version * 2 + (sh.split ? 1 : 0)) {
            case 10: go(wkv_kernel<5, false, true>); break;
            case 11: go(wkv_kernel<5, true, true>); break;
            case 12: go(wkv_kernel<6, false, true>); break;
            case 13: go(wkv_kernel<6, true, true>); break;
            case 14: go(wkv_kernel<7, false, true>); break;
            default: go(wkv_kernel<7, true, true>); break;
        }
        return;
    }
    switch (wp.version * 2 + (sh.split ? 1 : 0)) {
        case 10: launch_k(wkv_kernel<5>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
        case 11: launch_k(wkv_kernel<5, true>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
        case 12: launch_k(wkv_kernel<6>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
        case 13: launch_k(wkv_kernel<6, true>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
        case 14: launch_k(wkv_kernel<7>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
        default: launch_k(wkv_kernel<7, true>, grid, dim3(WKV_SA_THREADS), sm_b, wp, KC_WKV, s, prof, rows); break;
    }
}

// static split-K factor of a row-parallel projection: the S <= 8 / world (partial buffers the LN stages sum) that cuts K
// into whole 128-wide blocks, gives every CTA whole tiles and puts the most SMs to work.  (Measured, round 2: with the
// old cap of 4 the 3B channel-mix value projection ran on 40 CTAs, 22 us for 43 MB; 7 slices -> 140 CTAs.)
int b200rwkv_engine::pick_split(int K, int tiles) const {
    const int kb = K / GEMM_BK;
    if (K % GEMM_BK != 0) return 1;
    int best = 1;
    for (int S = 2; S <= 8 / world; ++S)
        if (kb % S == 0 && tiles * S <= num_sms) best = S;
    return best;
}

// dynamic shared memory limits of every projection kernel launch_gemm can pick (the quantised ones only for quantised plans)
static void gemm_smem_limits(int qtype) {
    CK(cudaFuncSetAttribute(gemm_kernel<1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<1, 2>::SMEM_BYTES));
    CK(cudaFuncSetAttribute(gemm_kernel<2, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<2, 2>::SMEM_BYTES));
    CK(cudaFuncSetAttribute(gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<2>::SMEM_BYTES));
    CK(cudaFuncSetAttribute(gemm_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<4>::SMEM_BYTES));
    CK(cudaFuncSetAttribute(gemm_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<8>::SMEM_BYTES));
    if (qtype == QT_INT8 || qtype == QT_NF4) {
#define QATTR(MT_, QT_)                                                                                                   \
    CK(cudaFuncSetAttribute(qgemm_kernel<MT_, QT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, QGemmCfg<MT_, QT_>::SMEM_BYTES)); \
    CK(cudaFuncSetAttribute(qgemm_tail_kernel<MT_, QT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, QGemmCfg<MT_, QT_>::SMEM_BYTES))
        QATTR(1, QT_INT8); QATTR(2, QT_INT8); QATTR(4, QT_INT8); QATTR(8, QT_INT8);
        QATTR(1, QT_NF4); QATTR(2, QT_NF4); QATTR(4, QT_NF4); QATTR(8, QT_NF4);
#undef QATTR
    }
    if (qtype == QT_FP8) {
        CK(cudaFuncSetAttribute(fp8gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<1>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<2>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<4>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<8>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_tail_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<1, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_tail_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<2, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_tail_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<4, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(fp8gemm_tail_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8GemmCfg<8, true>::SMEM_BYTES));
    }
    if (qtype == QT_INT4) {
        CK(cudaFuncSetAttribute(int4gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<1>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<2>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<4>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<8>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_tail_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<1, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_tail_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<2, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_tail_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<4, true>::SMEM_BYTES));
        CK(cudaFuncSetAttribute(int4gemm_tail_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Int4GemmCfg<8, true>::SMEM_BYTES));
    }
}

// dynamic shared memory limit of every WKV kernel launch_wkv can pick: prefill steps of up to 128 tokens, the decay-LoRA slice
// of the v6 fold and the staged rows live there
static void wkv_smem_limits() {
    const int wkv_smem_max = 96 * 1024;
    CK(cudaFuncSetAttribute(wkv_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<5, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<6, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<7, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<5, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<6, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<7, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<5, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<6, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
    CK(cudaFuncSetAttribute(wkv_kernel<7, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wkv_smem_max));
}

// k-major copy of the time_decay_w2 rows c0 .. c0 + 64 Hl - 1 (w2: [C][Dd] f16 as stored), one contiguous [Dd][64] slice per
// head: the operand of the v6 decay fold inside the WKV kernel
static std::vector<__half> wd2_k_major(const __half* w2, int c0, int Hl, int Dd) {
    std::vector<__half> t((size_t)Hl * Dd * 64);
    for (int h = 0; h < Hl; ++h)
        for (int k = 0; k < Dd; ++k)
            for (int c = 0; c < 64; ++c) t[((size_t)h * Dd + k) * 64 + c] = w2[(size_t)(c0 + h * 64 + c) * Dd + k];
    return t;
}

// One fill from its tensor's f16 values at `src` (device), on the engine's stream with the build's launch shapes.
void b200rwkv_engine::run_fill(const Fill& f, const __half* src, cudaStream_t s) {
    switch (f.kind) {
        case FILL_SEG: {
            const __half* m = src + f.off;
            uint8_t* dst = static_cast<uint8_t*>(f.dst);
            if (f.qtype == QT_NONE) {
                launch_repack(num_sms, m, f.ld, f.n0, f.k0, f.N, f.K, reinterpret_cast<uint4*>(dst), s, f.dst_kb);
                return;
            }
            if (f.qtype == QT_FP8) {
                // one warp per row; the scale is the absmax of the whole source row, whichever k slice this segment holds
                const int grid = std::min(cdiv(f.tiles * GEMM_BN, 8), num_sms * 32);
                quantize_fp8_kernel<<<grid, 256, 0, s>>>(m, f.ld, f.n0, f.k0, f.N, f.tiles, f.kb, dst, f.scales);
            } else {
                const size_t nwarp = (size_t)f.tiles * f.kb * GEMM_BN;
                const int grid = (int)std::min<size_t>((nwarp + 7) / 8, (size_t)num_sms * 32);
                if (f.qtype == QT_INT8) quantize_weight_kernel<QT_INT8><<<grid, 256, 0, s>>>(m, f.ld, f.n0, f.k0, f.N, f.tiles, f.kb, dst);
                else if (f.qtype == QT_INT4) quantize_int4_kernel<<<grid, 256, 0, s>>>(m, f.ld, f.n0, f.k0, f.N, f.tiles, f.kb, dst);
                else quantize_weight_kernel<QT_NF4><<<grid, 256, 0, s>>>(m, f.ld, f.n0, f.k0, f.N, f.tiles, f.kb, dst);
            }
            CK(cudaGetLastError());
            return;
        }
        case FILL_VEC: launch_f16_to_f32(src + f.off, static_cast<float*>(f.dst), f.count, f.scale, f.bias, s); return;
        case FILL_DECAY: launch_decay_table(src + f.off, static_cast<float*>(f.dst), (int)f.count, s); return;
        case FILL_RAW: CK(cudaMemcpyAsync(f.dst, src, f.count * 2, cudaMemcpyDeviceToDevice, s)); return;
        case FILL_FOLD: {
            std::vector<__half> rows((size_t)C * f.K);
            CK(cudaMemcpyAsync(rows.data(), src, rows.size() * 2, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            const std::vector<__half> t = wd2_k_major(rows.data(), f.n0, f.N, f.K);
            CK(cudaMemcpyAsync(f.dst, t.data(), t.size() * 2, cudaMemcpyHostToDevice, s));
            CK(cudaStreamSynchronize(s));        // `t` goes out of scope
            return;
        }
        default: throw Error(B200RWKV_ERR_INVALID, "internal: fill kind");
    }
}

// Every fill of each tensor of `in`, reading its values as F16 from d_tmp (grown to the largest tensor; the caller releases
// it): an image's bytes are copied up (and LoRA files blended in at creation), device tensors converted with round-to-nearest
// -even.  time_state is read on the host as F16, BF16 or F32, as creation reads it.  All on the engine's stream, complete on
// return.  The caller has checked every name, dtype and shape.
void b200rwkv_engine::fill_weights(const std::vector<WeightIn>& in) {
    size_t need = 16;
    for (const WeightIn& w : in) need = std::max(need, (size_t)w.numel * 2);
    d_tmp.grow(need, need);
    cudaStream_t s = stream;
    for (const WeightIn& w : in) {
        auto it = fills.find(w.name);
        if (it == fills.end()) continue;           // a tensor of the model the engine does not read
        if (it->second.front().kind == FILL_INIT) {
            StTensor t;
            std::vector<uint8_t> bytes;
            if (w.host) t = *w.host;
            else {
                const size_t esz = w.dtype == B200RWKV_DTYPE_F32 ? 4 : 2;
                bytes.resize((size_t)w.numel * esz);
                CK(cudaMemcpyAsync(bytes.data(), w.dev, bytes.size(), cudaMemcpyDeviceToHost, s));
                CK(cudaStreamSynchronize(s));
                t.dtype = w.dtype == B200RWKV_DTYPE_F32 ? "F32" : w.dtype == B200RWKV_DTYPE_BF16 ? "BF16" : "F16";
                t.data = bytes.data();
                t.nbytes = bytes.size();
            }
            if (init_state.empty()) init_state.assign((size_t)L * (N + 2) * C, 0.f);
            for (const Fill& f : it->second) time_state_rows(t, f.layer, H, N, C, init_state);
            continue;
        }
        if (w.host) {
            CK(cudaMemcpyAsync(d_tmp, w.host->data, w.host->nbytes, cudaMemcpyHostToDevice, s));
            if (!loras.empty()) {
                CK(cudaStreamSynchronize(s));
                blend_loras(*w.host);              // synchronises the device
            }
        } else if (w.dtype == B200RWKV_DTYPE_F16) {
            CK(cudaMemcpyAsync(d_tmp, w.dev, (size_t)w.numel * 2, cudaMemcpyDeviceToDevice, s));
        } else {
            const int grid = (int)std::min<size_t>(((size_t)w.numel + 255) / 256, (size_t)num_sms * 16);
            if (w.dtype == B200RWKV_DTYPE_F32) to_f16_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(w.dev), d_tmp, w.numel);
            else to_f16_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(w.dev), d_tmp, w.numel);
            CK(cudaGetLastError());
        }
        for (const Fill& f : it->second) run_fill(f, d_tmp, s);     // the next tensor's copy into d_tmp waits on the stream
    }
    CK(cudaStreamSynchronize(s));
}

// -----------------------------------------------------------------------------------------
// model build
// -----------------------------------------------------------------------------------------
void b200rwkv_engine::build(const StFile& st) {
    info = derive_info(st);
    check_loras(st);
    L = info.num_layer; C = info.num_emb; F = info.num_hidden; V = info.num_vocab; H = info.num_head; N = info.head_size;
    REQUIRE(N == 64, B200RWKV_ERR_UNSUPPORTED, "head_size must be 64");
    REQUIRE(H * N == C, B200RWKV_ERR_UNSUPPORTED, "num_head * head_size must equal num_emb");
    REQUIRE(C % 64 == 0 && C <= 8192, B200RWKV_ERR_UNSUPPORTED, "num_emb must be a multiple of 64 and <= 8192");
    REQUIRE(H % world == 0 && F % (8 * world) == 0 && V % world == 0, B200RWKV_ERR_UNSUPPORTED,
            "heads / hidden / vocab do not shard evenly over the tensor-parallel world");
    Cl = C / world; Hl = H / world; Fl = F / world; Vl = V / world;
    const int ver = info.version;
    const int c0 = rank * Cl, f0 = rank * Fl, v0 = rank * Vl;

    stream = new_stream();
    sm_stream = new_stream();
    if (quant_layers > 0 && quant_type != QT_NONE) {
        REQUIRE(quant_type == QT_INT8 || quant_type == QT_NF4 || quant_type == QT_FP8 || quant_type == QT_INT4, B200RWKV_ERR_UNSUPPORTED,
                "quant_type must be Int8, NF4, FP8 or Int4 (SF4 is not implemented)");
        REQUIRE(world == 1, B200RWKV_ERR_UNSUPPORTED, "quantised layers are single-GPU in this version");
        REQUIRE(precision == 0, B200RWKV_ERR_UNSUPPORTED, "quantised layers run with precision 0 (f16 operands)");
    }
    gemm_smem_limits(quant_layers > 0 ? quant_type : (int)QT_NONE);
    wkv_smem_limits();
    if (precision == 1) split_act = true;         // f32-activation mode (web-rwkv `Bundle::<f32>`): no activation is rounded to f16

    // ---- step metadata ----
    meta_ints = MetaView::ints(maxT, S);
    d_meta = (int*)dalloc(meta_ints * 4);
    h_meta = HostBuf<int>(meta_ints * 4 * META_RING);
    memset(h_meta, 0, meta_ints * 4 * META_RING);
    for (auto& ev : meta_ev) ev = new_event(cudaEventDisableTiming);
    MetaView mv{d_meta, maxT, S};

    // ---- state ----
    att_shift = (float*)dalloc((size_t)L * S * C * 4);
    ffn_shift = (float*)dalloc((size_t)L * S * C * 4);
    wkv_state = (float*)dalloc((size_t)L * S * Hl * N * N * 4);
    d_api = (float*)dalloc((size_t)L * (N + 2) * C * 4);
    // State::init() with a state-tuned model (FILL_INIT rows); empty otherwise
    {
        std::vector<float> probe;
        if (state_from_st(st, L, H, N, C, probe))
            for (int l = 0; l < L; ++l) {
                Fill f;
                f.kind = FILL_INIT; f.layer = l;
                fills["blocks." + std::to_string(l) + ".att.time_state"].push_back(f);
            }
    }

    // ---- activations ----
    const size_t TC = (size_t)maxT * C, TCl = (size_t)maxT * Cl;
    x_a = (float*)dalloc(TC * 4); x_b = (float*)dalloc(TC * 4);
    xx1 = (float*)dalloc(TC * 4); sx1 = (float*)dalloc(TC * 4); xx2 = (float*)dalloc(TC * 4);
    f_r = (float*)dalloc(TCl * 4); f_k = (float*)dalloc(TCl * 4); f_v = (float*)dalloc(TCl * 4); f_g = (float*)dalloc(TCl * 4);
    f_w = (float*)dalloc(TCl * 4); f_a = (float*)dalloc(TCl * 4); f_nu = (float*)dalloc(TCl * 4); f_vfirst = (float*)dalloc(TCl * 4);
    {
        auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
        off_part_att = 0;
        off_part_ffn = al(off_part_att + TC * 4 * 8);       // up to 8 split-K slices each
        off_rr = al(off_part_ffn + TC * 4 * 8);
        off_logits = al(off_rr + TCl * 4);
        off_flags = al(off_logits + (size_t)maxT * Vl * 4);
        comm_bytes = al(off_flags + 256);
        comm_base = (uint8_t*)dalloc(comm_bytes, true);
        part_att = (float*)(comm_base + off_part_att);
        part_ffn = (float*)(comm_base + off_part_ffn);
        f_rr = (float*)(comm_base + off_rr);
        d_logits = (float*)(comm_base + off_logits);
        d_epoch = (unsigned*)dalloc(16, true);
        pre_gbar = (unsigned*)dalloc(256, true);
        ln_cluster_ok = ln_cluster_fits(C);
        split_on = split_act && ln_cluster_ok;
        REQUIRE(precision != 1 || split_on, B200RWKV_ERR_UNSUPPORTED, "precision 1 needs num_emb to be a multiple of 32 and <= 8192");
    }
    const int S_att = pick_split(Cl, cdiv(C, GEMM_BN)), S_ffn = pick_split(Fl, cdiv(C, GEMM_BN));
    split_att = S_att; split_ffn = S_ffn;
    d_hidden = (float*)dalloc(TC * 4);
    d_hid_tab = (float**)dalloc((size_t)L * sizeof(float*));
    step_done = new_event(cudaEventDisableTiming);
    keep_valid.assign(S, 0);
    if (rank == 0) {
        d_keep = (float*)dalloc((size_t)S * V * 4);
        const int nseg = cdiv(V, TOPK_SEG);
        if (nseg <= TOPK_MAX_SEGS) {       // larger vocabularies: b200rwkv_sample_topk answers UNSUPPORTED
            tk_cand_x = (float*)dalloc((size_t)S * nseg * TOPK_MAX * 4);
            tk_cand_id = (unsigned*)dalloc((size_t)S * nseg * TOPK_MAX * 4);
            tk_stats = (float2*)dalloc((size_t)S * nseg * 8);
            tk_out_id = (unsigned*)dalloc((size_t)S * TOPK_MAX * 4);
            tk_out_p = (float*)dalloc((size_t)S * TOPK_MAX * 4);
        }
    }
    // with adapters, every projection operand carries one 128-wide tail block per adapter after its own k blocks
    auto op_cols = [&](int K) { return n_adapters ? (cdiv(K, GEMM_BK) + n_adapters) * GEMM_BK : K; };
    for (int i = 0; i < 6; ++i) a_x[i] = a16_alloc(op_cols(C));
    a_out = a16_alloc(op_cols(Cl));
    a_kk = a16_alloc(op_cols(Fl));
    a_head = a16_alloc(op_cols(C));
    slot_adapter.assign(S, 0);
    if (n_adapters) d_slot_adapter = (int*)dalloc((size_t)S * 4, true);

    // ---- embedding + ln0 ----
    {
        const StTensor& e = st.get("emb.weight");
        emb = (__half*)dalloc(e.nbytes, false);
        Fill f;
        f.kind = FILL_RAW; f.count = (size_t)e.numel(); f.dst = emb;
        fills[e.name].push_back(f);
        embed.emb = emb; embed.C = C; embed.V = V; embed.meta = mv;
        embed.ln_w = vec_f32(st, "blocks.0.ln0.weight", 0, C);
        embed.ln_b = vec_f32(st, "blocks.0.ln0.bias", 0, C);
        embed.x_out = x_a;
    }

    // step-shape fields (kq_tile, d1_kq, an A16 ldo) stay 0 here: the launch_* functions fill them in per step
    auto base_ln = [&](LnMixParams& p) {
        memset(&p, 0, sizeof(p));
        p.C = C; p.meta = mv;
    };
    auto f32_seg = [&](const StTensor& t, int n0, int Nn, int k0, int K, const A16Buf& ab, float* out, int ldo, int act,
                       const float* bias, int a_koff = 0, int a_mat = 0) {
        SegDesc d;
        d.t = &t; d.n0 = n0; d.N = Nn; d.k0 = k0; d.K = K;
        REQUIRE(a_koff % GEMM_BK == 0, B200RWKV_ERR_INVALID, "internal: split-K slices start on k-block boundaries");
        d.proto.A = ab.p + (size_t)a_mat * ab.halves_per_matrix + (size_t)(a_koff / GEMM_BK) * A16_KB_HALVES;
        d.proto.out_mode = OUT_F32; d.proto.act = act; d.proto.bias = bias; d.proto.out = out; d.proto.ldo = ldo;
        return d;
    };
    auto a16_seg = [&](const StTensor& t, int n0, int Nn, int k0, int K, const A16Buf& ab, const A16Buf& dst, int act,
                       const float* bias) {
        SegDesc d;
        d.t = &t; d.n0 = n0; d.N = Nn; d.k0 = k0; d.K = K;
        d.proto.A = ab.p;
        d.proto.out_mode = OUT_A16; d.proto.act = act; d.proto.bias = bias; d.proto.out = dst.p;
        return d;
    };

    layers.resize(L);
    for (int l = 0; l < L; ++l) {
        Layer& ly = layers[l];
        const std::string b = "blocks." + std::to_string(l) + ".";
        const std::string a = b + "att.", f = b + "ffn.";
        float* att_sh = att_shift + (size_t)l * S * C;
        float* ffn_sh = ffn_shift + (size_t)l * S * C;
        // `quant`: the eight projection matrices of the first layers are quantised, adapters / LoRA matrices stay f16 -- so a
        // launch that mixed both kinds (R/K/V/G + decay LoRA, v7 R/K/V + adapters) goes out as two in those layers
        const int lq = (l < quant_layers) ? quant_type : QT_NONE;

        // ---------------- LN1 (+ residual update from the previous layer's channel mix, wired by finalize_tp) ----------------
        LnMixParams& n1 = ly.ln1;
        base_ln(n1);
        n1.x_in = (l == 0) ? x_a : x_b;
        n1.x_out = x_a;
        if (l > 0) {
            n1.commit_dst = ffn_shift + (size_t)(l - 1) * S * C;
            n1.commit_src = xx2;
            n1.hid_slot = d_hid_tab + (l - 1);       // x_out here is the residual stream after layer l - 1
        }
        n1.ln_w = vec_f32(st, b + "ln1.weight", 0, C);
        n1.ln_b = vec_f32(st, b + "ln1.bias", 0, C);
        n1.shift_state = att_sh;
        n1.xx_out = xx1;

        WkvParams& wk = ly.wkv;
        memset(&wk, 0, sizeof(wk));
        wk.version = ver; wk.ld = Cl; wk.meta = mv; wk.H = Hl;
        wk.state = wkv_state + (size_t)l * S * Hl * N * N;
        wk.r = f_r; wk.k = f_k; wk.v = f_v; wk.g = f_g;
        wk.lnx_w = vec_f32(st, a + "ln_x.weight", c0, Cl);
        wk.lnx_b = vec_f32(st, a + "ln_x.bias", c0, Cl);
        wk.out = a_out.p;

        const StTensor& Wr = st.get(a + "receptance.weight");
        const StTensor& Wk = st.get(a + "key.weight");
        const StTensor& Wv = st.get(a + "value.weight");
        const StTensor& Wo = st.get(a + "output.weight");

        if (ver == 6) {
            const int Dm = info.time_mix_adapter, Dd = info.time_decay_adapter;
            if (l == 0) {
                a_lora[0] = a16_alloc(Dm, 5);   // tanh(W1 xxx), five groups
                a_lora[1] = a16_alloc(Dd);      // tanh(Wd1 xw)
            }
            n1.n_mix = 1;
            n1.mu[0] = vec_f32(st, a + "time_mix_x", 0, C);
            n1.mix_out[0] = a_x[5].p;           // xxx
            n1.sx_out = sx1;
            // W1: [5*Dm, C]
            {
                std::vector<SegDesc> sv;
                SegDesc d = a16_seg(st.get(a + "time_mix_w1"), 0, 5 * Dm, 0, C, a_x[5], a_lora[0], ACT_TANH, nullptr);
                d.proto.grp = Dm;
                d.proto.grp_stride = (int)a_lora[0].halves_per_matrix;
                sv.push_back(d);
                ly.lora.push_back(make_launch(sv));
            }
            // W2: [5, C, Dm]; order w,k,v,r,g (SURVEY.md App. A)
            static const char* names[5] = {"time_mix_w", "time_mix_k", "time_mix_v", "time_mix_r", "time_mix_g"};
            const float* mu5[5];
            for (int i = 0; i < 5; ++i) mu5[i] = vec_f32(st, a + names[i], 0, C);
            {
                std::vector<SegDesc> sv;
                for (int i = 0; i < 5; ++i) {
                    SegDesc d;
                    d.t = &st.get(a + "time_mix_w2"); d.slice = i; d.n0 = 0; d.N = C; d.k0 = 0; d.K = Dm;
                    d.proto.A = a_lora[0].p + (size_t)i * a_lora[0].halves_per_matrix;
                    d.proto.out_mode = OUT_LERP_A16; d.proto.act = ACT_NONE;
                    d.proto.out = a_x[i].p;
                    d.proto.aux0 = xx1; d.proto.aux1 = sx1; d.proto.aux2 = mu5[i]; d.proto.ld_aux = C;
                    sv.push_back(d);
                }
                ly.lora.push_back(make_launch(sv));
            }
            {   // the raw copies below are indexed with these exact shapes
                const StTensor& w1 = st.get(a + "time_mix_w1");
                const StTensor& w2 = st.get(a + "time_mix_w2");
                const StTensor& d2 = st.get(a + "time_decay_w2");
                REQUIRE(w1.shape.size() == 2 && w1.shape[0] == 5 * Dm && w1.shape[1] == C, B200RWKV_ERR_INVALID, "time_mix_w1 must be [5*Dm, C]");
                REQUIRE(w2.shape.size() == 3 && w2.shape[0] == 5 && w2.shape[1] == C && w2.shape[2] == Dm, B200RWKV_ERR_INVALID,
                        "time_mix_w2 must be [5, C, Dm]");
                REQUIRE(d2.shape.size() == 2 && d2.shape[0] == C && d2.shape[1] == Dd, B200RWKV_ERR_INVALID, "time_decay_w2 must be [C, Dd]");
            }
            if (pre6_fits(Dm, C)) {
                auto upload_raw = [&](const StTensor& t) {
                    Fill f;
                    f.kind = FILL_RAW; f.count = (size_t)t.numel(); f.dst = dalloc(t.nbytes, false);
                    fills[t.name].push_back(f);
                    return (__half*)f.dst;
                };
                Pre6Params& q = ly.pre6;
                q.W1 = upload_raw(st.get(a + "time_mix_w1"));     // row-major copies of the ddlerp LoRA weights
                q.W2 = upload_raw(st.get(a + "time_mix_w2"));
                for (int i = 0; i < 5; ++i) { q.mu[i] = mu5[i]; q.out[i] = a_x[i].p; }
                q.lora = a_lora[0].p; q.lora_stride = (int)a_lora[0].halves_per_matrix;
                q.Dm = Dm;
                q.gbar = pre_gbar;
                ly.has_pre6 = true;
            }
            // R,K,V,G (column parallel by head) + decay LoRA stage 1 (replicated)
            {
                std::vector<SegDesc> sv;
                sv.push_back(f32_seg(Wr, c0, Cl, 0, C, a_x[3], f_r, Cl, ACT_NONE, nullptr));
                sv.push_back(f32_seg(Wk, c0, Cl, 0, C, a_x[1], f_k, Cl, ACT_NONE, nullptr));
                sv.push_back(f32_seg(Wv, c0, Cl, 0, C, a_x[2], f_v, Cl, ACT_NONE, nullptr));
                sv.push_back(f32_seg(st.get(a + "gate.weight"), c0, Cl, 0, C, a_x[4], f_g, Cl, ACT_SILU, nullptr));
                if (lq != QT_NONE) {
                    // the small f16 launch goes first: it occupies a handful of SMs, and behind it the quantised launch is
                    // already resident on the others filling its ring (programmatic dependent launch)
                    std::vector<SegDesc> sd;
                    sd.push_back(a16_seg(st.get(a + "time_decay_w1"), 0, Dd, 0, C, a_x[0], a_lora[1], ACT_TANH, nullptr));
                    ly.pre.push_back(make_launch(sd));
                    ly.pre.push_back(make_launch(sv, 0, lq));
                } else {
                    sv.push_back(a16_seg(st.get(a + "time_decay_w1"), 0, Dd, 0, C, a_x[0], a_lora[1], ACT_TANH, nullptr));
                    ly.pre.push_back(make_launch(sv));
                }
            }
            // decay LoRA stage 2: w = exp(-exp(time_decay + Wd2 d))
            const float* time_decay = vec_f32(st, a + "time_decay", c0, Cl);
            if (Dd <= 128 && Dd % 8 == 0) {
                // k-major copy of this rank's time_decay_w2 rows, one contiguous [Dd][64] slice per head: the WKV
                // kernels evaluate the decay LoRA stage 2 themselves (one launch / phase less per layer)
                Fill fd;
                fd.kind = FILL_FOLD; fd.n0 = c0; fd.N = Hl; fd.K = Dd;
                fd.dst = dalloc((size_t)Hl * Dd * 64 * 2, false);
                fills[a + "time_decay_w2"].push_back(fd);
                wk.wd2t = (__half*)fd.dst;
                wk.decay_bias = time_decay;
                wk.d1 = a_lora[1].p;
                wk.Dd = Dd;
            } else {
                std::vector<SegDesc> sv;
                sv.push_back(f32_seg(st.get(a + "time_decay_w2"), c0, Cl, 0, Dd, a_lora[1], f_w, Cl, ACT_EXPNEGEXP, time_decay));
                ly.pre.push_back(make_launch(sv));
            }
            wk.w = f_w;
            wk.u = vec_f32(st, a + "time_first", c0, Cl);
        } else if (ver == 5) {
            // x_* = xx*mix + prev*(1-mix) == xx + (prev-xx)*(1-mix)
            static const char* names[4] = {"time_mix_k", "time_mix_v", "time_mix_r", "time_mix_g"};
            n1.n_mix = 4;
            for (int i = 0; i < 4; ++i) {
                n1.mu[i] = vec_f32(st, a + names[i], 0, C, -1.f, 1.f);
                n1.mix_out[i] = a_x[1 + i].p;     // k,v,r,g -> a_x[1..4]
            }
            std::vector<SegDesc> sv;
            sv.push_back(f32_seg(Wr, c0, Cl, 0, C, a_x[3], f_r, Cl, ACT_NONE, nullptr));
            sv.push_back(f32_seg(Wk, c0, Cl, 0, C, a_x[1], f_k, Cl, ACT_NONE, nullptr));
            sv.push_back(f32_seg(Wv, c0, Cl, 0, C, a_x[2], f_v, Cl, ACT_NONE, nullptr));
            sv.push_back(f32_seg(st.get(a + "gate.weight"), c0, Cl, 0, C, a_x[4], f_g, Cl, ACT_SILU, nullptr));
            ly.pre.push_back(make_launch(sv, 0, lq));
            {
                const StTensor& td = st.get(a + "time_decay");
                REQUIRE(td.numel() == C, B200RWKV_ERR_UNSUPPORTED, "v5 time_decay must be [H, N]");
                Fill f;
                f.kind = FILL_DECAY; f.off = (size_t)c0; f.count = (size_t)Cl; f.dst = dalloc((size_t)Cl * 4, false);
                fills[td.name].push_back(f);
                wk.w_static = (float*)f.dst;
            }
            wk.u = vec_f32(st, a + "time_first", c0, Cl);
        } else {
            // v7: six static lerps r,w,k,v,a,g -> a_x[0..5]
            static const char* names[6] = {"x_r", "x_w", "x_k", "x_v", "x_a", "x_g"};
            const int Dw = (int)st.dim(a + "w1", 0, 2), Da = (int)st.dim(a + "a1", 0, 2), Dg = (int)st.dim(a + "g1", 0, 2);
            const std::string v1n = L > 1 ? "blocks.1.att.v1" : "blocks.0.att.v1";
            const int Dv = st.find(v1n) ? (int)st.dim(v1n, 0, 2) : 32;
            if (l == 0) {
                a_lora[0] = a16_alloc(Dw); a_lora[1] = a16_alloc(Da); a_lora[2] = a16_alloc(Dv); a_lora[3] = a16_alloc(Dg);
            }
            n1.n_mix = 6;
            for (int i = 0; i < 6; ++i) {
                n1.mu[i] = vec_f32(st, a + names[i], 0, C);
                n1.mix_out[i] = a_x[i].p;
            }
            {
                std::vector<SegDesc> sv;
                sv.push_back(f32_seg(Wr, c0, Cl, 0, C, a_x[0], f_r, Cl, ACT_NONE, nullptr));
                sv.push_back(f32_seg(Wk, c0, Cl, 0, C, a_x[2], f_k, Cl, ACT_NONE, nullptr));
                sv.push_back(f32_seg(Wv, c0, Cl, 0, C, a_x[3], f_v, Cl, ACT_NONE, nullptr));
                std::vector<SegDesc> sq;
                if (lq != QT_NONE) sq.swap(sv);          // quantised R/K/V go out as their own launch, after the f16 adapters
                sv.push_back(a16_seg(st.get(a + "w1"), 0, Dw, 0, C, a_x[1], a_lora[0], ACT_TANH, nullptr));
                sv.push_back(a16_seg(st.get(a + "a1"), 0, Da, 0, C, a_x[4], a_lora[1], ACT_NONE, nullptr));
                if (l > 0) sv.push_back(a16_seg(st.get(a + "v1"), 0, Dv, 0, C, a_x[3], a_lora[2], ACT_NONE, nullptr));
                sv.push_back(a16_seg(st.get(a + "g1"), 0, Dg, 0, C, a_x[5], a_lora[3], ACT_SIGMOID, nullptr));
                ly.pre.push_back(make_launch(sv));
                if (lq != QT_NONE) ly.pre.push_back(make_launch(sq, 0, lq));
            }
            {
                std::vector<SegDesc> sv;
                sv.push_back(f32_seg(st.get(a + "w2"), c0, Cl, 0, Dw, a_lora[0], f_w, Cl, ACT_V7DECAY, vec_f32(st, a + "w0", c0, Cl)));
                sv.push_back(f32_seg(st.get(a + "a2"), c0, Cl, 0, Da, a_lora[1], f_a, Cl, ACT_SIGMOID, vec_f32(st, a + "a0", c0, Cl)));
                if (l > 0)
                    sv.push_back(f32_seg(st.get(a + "v2"), c0, Cl, 0, Dv, a_lora[2], f_nu, Cl, ACT_SIGMOID, vec_f32(st, a + "v0", c0, Cl)));
                sv.push_back(f32_seg(st.get(a + "g2"), c0, Cl, 0, Dg, a_lora[3], f_g, Cl, ACT_NONE, nullptr));
                ly.pre.push_back(make_launch(sv));
            }
            wk.w = f_w; wk.a = f_a; wk.nu = f_nu; wk.v_first = f_vfirst; wk.layer0 = (l == 0);
            wk.k_k = vec_f32(st, a + "k_k", c0, Cl);
            wk.k_a = vec_f32(st, a + "k_a", c0, Cl);
            wk.r_k = vec_f32(st, a + "r_k", c0, Cl);
        }

        // ---------------- output projection (row parallel) -> partial ----------------
        {
            // row-parallel: K is cut into `S_att` static slices, one partial buffer each (summed by the
            // next LN stage in fixed order); with tiles * S CTAs every CTA owns whole tiles: no fix-up
            std::vector<SegDesc> sv;
            for (int sp = 0; sp < S_att; ++sp)
                sv.push_back(f32_seg(Wo, 0, C, c0 + sp * (Cl / S_att), Cl / S_att, a_out, part_att + (size_t)sp * TC, C, ACT_NONE,
                                     nullptr, sp * (Cl / S_att)));
            ly.o = make_launch(sv, S_att > 1 ? cdiv(C, GEMM_BN) * S_att : 0, lq);
        }

        // ---------------- LN2 ----------------
        LnMixParams& n2 = ly.ln2;
        base_ln(n2);
        n2.x_in = x_a; n2.x_out = x_b;
        n2.ln_w = vec_f32(st, b + "ln2.weight", 0, C);
        n2.ln_b = vec_f32(st, b + "ln2.bias", 0, C);
        n2.shift_state = ffn_sh;
        n2.xx_out = xx2;
        n2.commit_dst = att_sh; n2.commit_src = xx1;
        const StTensor& Fk = st.get(f + "key.weight");
        const StTensor& Fv = st.get(f + "value.weight");
        if (ver == 7) {
            n2.n_mix = 1;
            n2.mu[0] = vec_f32(st, f + "x_k", 0, C);
            n2.mix_out[0] = a_x[0].p;
            std::vector<SegDesc> sv;
            sv.push_back(a16_seg(Fk, f0, Fl, 0, C, a_x[0], a_kk, ACT_RELU2, nullptr));
            ly.ffn.push_back(make_launch(sv, 0, lq));
        } else {
            n2.n_mix = 2;
            if (ver == 6) {
                n2.mu[0] = vec_f32(st, f + "time_mix_k", 0, C);
                n2.mu[1] = vec_f32(st, f + "time_mix_r", 0, C);
            } else {
                n2.mu[0] = vec_f32(st, f + "time_mix_k", 0, C, -1.f, 1.f);
                n2.mu[1] = vec_f32(st, f + "time_mix_r", 0, C, -1.f, 1.f);
            }
            n2.mix_out[0] = a_x[0].p;
            n2.mix_out[1] = a_x[1].p;
            std::vector<SegDesc> sv;
            sv.push_back(a16_seg(Fk, f0, Fl, 0, C, a_x[0], a_kk, ACT_RELU2, nullptr));
            sv.push_back(f32_seg(st.get(f + "receptance.weight"), c0, Cl, 0, C, a_x[1], f_rr, Cl, ACT_SIGMOID, nullptr));
            ly.ffn.push_back(make_launch(sv, 0, lq));
        }
        {
            std::vector<SegDesc> sv;
            for (int sp = 0; sp < S_ffn; ++sp)
                sv.push_back(f32_seg(Fv, 0, C, f0 + sp * (Fl / S_ffn), Fl / S_ffn, a_kk, part_ffn + (size_t)sp * TC, C, ACT_NONE,
                                     nullptr, sp * (Fl / S_ffn)));
            ly.ffn.push_back(make_launch(sv, S_ffn > 1 ? cdiv(C, GEMM_BN) * S_ffn : 0, lq));
        }
    }

    // ---------------- ln_out + head ----------------
    memset(&lnout, 0, sizeof(lnout));
    lnout.x_in = x_b; lnout.C = C; lnout.meta = mv;
    lnout.ln_w = vec_f32(st, "ln_out.weight", 0, C);
    lnout.ln_b = vec_f32(st, "ln_out.bias", 0, C);
    lnout.head_in = a_head.p;
    lnout.commit_dst = ffn_shift + (size_t)(L - 1) * S * C;
    lnout.commit_src = xx2;
    lnout.hidden_out = d_hidden;
    {
        std::vector<SegDesc> sv;
        sv.push_back(f32_seg(st.get("head.weight"), v0, Vl, 0, C, a_head, d_logits, Vl, ACT_NONE, nullptr));
        head = make_launch(sv);
        head.p.nrows = d_meta + 2;    // R
    }

    // adapter plans: every launch that holds an adapted projection again as W', with a shrink launch in front of it
    if (n_adapters) {
        ad_layers.resize(L);
        auto shrink = [&](AdapterParams& sp, bool on_head) {
            memset(&sp, 0, sizeof(sp));
            sp.n = n_adapters; sp.meta = mv; sp.slot_adapter = d_slot_adapter; sp.head = on_head ? 1 : 0;
        };
        for (int l = 0; l < L; ++l) {
            Layer& ly = layers[l];
            AdLayer& ad = ad_layers[l];
            shrink(ad.s_pre, false); shrink(ad.s_o, false); shrink(ad.s_fk, false); shrink(ad.s_fv, false);
            for (auto& g : ly.pre) ad.pre.push_back(ad_launch(g, ad.s_pre));
            ad.o = ad_launch(ly.o, ad.s_o);
            REQUIRE(ly.ffn.size() == 2, B200RWKV_ERR_INVALID, "internal: channel mix is two launches");
            ad.ffn.push_back(ad_launch(ly.ffn[0], ad.s_fk));
            ad.ffn.push_back(ad_launch(ly.ffn[1], ad.s_fv));
        }
        shrink(s_head, true);
        ad_head = ad_launch(head, s_head);
        ad_head.p.nrows = d_meta + 2;
        if (ad_targets)
            REQUIRE(ad_mats.size() == ad_place_matrices(st.tensors, ad_targets, ad_quant_layers(), quant_type).size(),
                    B200RWKV_ERR_INVALID, "internal: a targeted matrix has no W' plan");
        // load_adapter's staging
        size_t cols = 0, blocks = 0;
        for (const AdMatrix& m : ad_mats) {
            cols = std::max(cols, (size_t)m.N * GEMM_BK * 2);
            blocks = std::max(blocks, (size_t)m.tiles * GEMM_WBYTES);
        }
        ad_stage_cols = cols;
        ad_stage = (uint8_t*)dalloc(cols + blocks, false);
        place_full.assign(n_adapters, adapters.empty() ? 0 : 1);
    }
    gemm_ws = (float*)dalloc(gemm_ws_floats * 4, false);
    auto wire = [&](GemmLaunch& g) {
        g.p.ws = gemm_ws;
        g.src.clear();          // points into the model file, which is borrowed during build only
    };
    for (auto& ly : layers) {
        for (auto& g : ly.lora) wire(g);
        for (auto& g : ly.pre) wire(g);
        wire(ly.o);
        for (auto& g : ly.ffn) wire(g);
    }
    wire(head);
    for (auto& ad : ad_layers) {
        for (auto& g : ad.pre) wire(g);
        wire(ad.o);
        for (auto& g : ad.ffn) wire(g);
    }
    wire(ad_head);

    if (world == 1) {
        peer_base[0] = comm_base;
        finalize_tp();
    }
    // the model's tensor names and shapes, for load_adapter's file checks and the weight updates' checks
    for (auto& kv : st.tensors) {
        StTensor t = kv.second;
        t.data = nullptr;
        model_shapes.emplace(kv.first, std::move(t));
    }
    had_loras = !loras.empty();
    // every weight fill, after the zeroing and the adapter data above (the legacy stream) have landed
    CK(cudaDeviceSynchronize());
    std::vector<WeightIn> in;
    for (auto& kv : fills) {
        const StTensor& t = st.tensors.at(kv.first);
        in.push_back({kv.first, &t, nullptr, B200RWKV_DTYPE_F16, t.numel()});
    }
    fill_weights(in);
    d_tmp = Buf<__half>();
}

// -----------------------------------------------------------------------------------------
// Tensor parallel wiring: every LN stage sums the partial projections of ALL ranks (rank-major,
// then split-K slice: the same fixed order on every rank, so the replicated residual stream stays
// bit-identical across ranks) straight out of the peers' comm blocks, and takes the channel-mix
// gate block-wise from the rank that owns those columns.
// -----------------------------------------------------------------------------------------
void b200rwkv_engine::finalize_tp() {
    const size_t TC = (size_t)maxT * C;
    const int ver = info.version;
    auto parts_of = [&](size_t off, int S, const float** dst) {
        int n = 0;
        for (int q = 0; q < world; ++q)
            for (int sp = 0; sp < S; ++sp) dst[n++] = (const float*)(peer_base[q] + off) + (size_t)sp * TC;
        return n;
    };
    auto gates_of = [&](const float** dst) {
        for (int q = 0; q < world; ++q) dst[q] = (const float*)(peer_base[q] + off_rr);
    };
    for (int l = 0; l < L; ++l) {
        Layer& ly = layers[l];
        if (l > 0) {
            ly.ln1.n_parts = parts_of(off_part_ffn, split_ffn, ly.ln1.parts);
            if (ver != 7) { ly.ln1.n_gate = world; ly.ln1.gate_cl = Cl; gates_of(ly.ln1.gates); }
        }
        ly.ln2.n_parts = parts_of(off_part_att, split_att, ly.ln2.parts);
    }
    lnout.n_parts = parts_of(off_part_ffn, split_ffn, lnout.parts);
    if (ver != 7) { lnout.n_gate = world; lnout.gate_cl = Cl; gates_of(lnout.gates); }
    memset(&tpbar, 0, sizeof(tpbar));
    for (int q = 0; q < world; ++q) tpbar.flags[q] = (unsigned*)(peer_base[q] + off_flags);
    tpbar.epoch = d_epoch;
    tpbar.rank = rank;
    tpbar.world = world;
    connected = true;
}

// [r][K] rows of A = lora.0^T ([in, r] on disk) for the shrink kernel: one 16-byte load per 8 k of a row
static std::vector<uint16_t> adapter_a_rows(const uint8_t* lora0, int K, int r) {
    // whole groups of 8 rows, zeros past r: the shrink kernel loads the 8 rows of its columns without a bound check
    std::vector<uint16_t> raw((size_t)K * r), rows((size_t)cdiv(r, 8) * 8 * K, 0);
    memcpy(raw.data(), lora0, raw.size() * 2);
    for (int k = 0; k < K; ++k)
        for (int j = 0; j < r; ++j) rows[(size_t)j * K + k] = raw[(size_t)k * r + j];
    return rows;
}

// The W' plan of `base` (one tail k block per adapter place on each segment that holds a whole planned projection, or the
// last split-K slice of one), with the projection added to the shrink launch `sp` and to ad_mats; `base` itself when no
// projection of it is planned.  Planned: a matrix some adapter file pairs, or on a places engine a targeted one (every
// place's A rows are reserved at the rank limit, so a later load_adapter allocates nothing).
GemmLaunch b200rwkv_engine::ad_launch(const GemmLaunch& base, AdapterParams& sp) {
    std::vector<SegDesc> segs = base.src;
    std::vector<AdMatrix> mats;
    std::vector<int> mat_seg;
    for (size_t i = 0; i < segs.size(); ++i) {
        SegDesc& d = segs[i];
        const StTensor& t = *d.t;
        if (d.slice >= 0 || !ends_with(t.name, ".weight") || t.shape.size() != 2 || d.k0 + d.K != t.shape[1]) continue;
        const std::string nm = t.name.substr(0, t.name.size() - 7);
        bool planned = (ad_target_bit(nm) & ad_targets) && !in_quant_layer(nm, ad_quant_layers(), quant_type);
        for (const LoraSrc& a : adapters) planned = planned || a.st->find(nm + ".lora.0");
        if (!planned) continue;
        REQUIRE((base.qtype == QT_NONE || quant_adapters) && world == 1 && d.k0 % GEMM_BK == 0 && sp.nproj < AD_MAX_PROJ, B200RWKV_ERR_INVALID,
                "internal: adapter on " + nm + " does not fit its launch");
        AdapterProj pj;
        memset(&pj, 0, sizeof(pj));
        pj.K = (int)t.shape[1];
        AdMatrix m{nm, d.N, pj.K, nullptr, 0, 0, 0, &sp, sp.nproj, {}};
        for (int a = 0; a < n_adapters; ++a) {
            m.A[a] = (__half*)dalloc((size_t)AD_MAX_RANK * pj.K * 2, true);
            pj.A[a] = m.A[a];
            const StTensor* la = a < (int)adapters.size() ? adapters[a].st->find(nm + ".lora.0") : nullptr;
            if (!la) continue;          // rank 0: the shrink writes zeros into this place's tail block
            pj.r[a] = (int)la->shape[1];
            const std::vector<uint16_t> rows = adapter_a_rows(la->data, pj.K, pj.r[a]);
            CK(cudaMemcpy(m.A[a], rows.data(), rows.size() * 2, cudaMemcpyHostToDevice));
        }
        pj.op = const_cast<__half*>(d.proto.A) - (size_t)(d.k0 / GEMM_BK) * A16_KB_HALVES;
        pj.kb0 = cdiv(pj.K, GEMM_BK);
        sp.p[sp.nproj++] = pj;
        d.ad_tail = n_adapters;
        mats.push_back(m);
        mat_seg.push_back((int)i);
    }
    if (mats.empty()) return base;
    // quantised: the codes are quantised from the same rows as the base plan's, so they are its codes
    GemmLaunch g = make_launch(segs, base.force_grid, base.qtype, B200RWKV_PLAN_ADAPTER);
    for (size_t j = 0; j < mats.size(); ++j) {
        const GemmSeg& sg = g.p.seg[mat_seg[j]];
        mats[j].tiles = sg.tiles;
        if (g.qtype == QT_NONE) {
            mats[j].W = (uint8_t*)g.p.W + (size_t)sg.blk_begin * GEMM_WBYTES;
            mats[j].KB = sg.KB;
            mats[j].kbw = sg.KB - n_adapters;
        } else {                        // the tail blocks alone: [tile][place]
            mats[j].W = const_cast<uint8_t*>(g.p.tails) + (size_t)g.p.tblk[mat_seg[j]] * GEMM_WBYTES;
            mats[j].KB = n_adapters;
            mats[j].kbw = 0;
        }
        ad_mats.push_back(mats[j]);
    }
    return g;
}

// Place `id`'s rank on one matrix, in the shrink launch that holds it (and its copy for the snapshot rows' head launch).
// Ranks are launch parameters: the caller drops the captured adapter step graphs.
void b200rwkv_engine::set_place_rank(const AdMatrix& m, int id, int r) {
    m.sp->p[m.proj].r[id - 1] = r;
    if (m.sp == &s_head && snap_dev) s_snap_head.p[m.proj].r[id - 1] = r;
}

// The step graphs captured with the adapter plans (key bit 128, snapshot variants included) hold the shrink parameters as
// they were; unbound steps keep theirs.
void b200rwkv_engine::drop_adapter_graphs() {
    for (auto it = graphs.begin(); it != graphs.end();) it = (it->first & 128) ? graphs.erase(it) : std::next(it);
}

// b200rwkv_load_adapter after its checks: into every planned matrix the file pairs, place `id`'s tail block of W' =
// f16(alpha lora.1) with zeros past the rank (make_launch's rounding, re-tiled by the load-time repack kernel), its A rows
// and its rank.  The place is empty, so the other matrices already hold zeros and rank 0.  Everything goes on the engine's
// stream (steps already enqueued finish with the old contents) and is complete on return.
void b200rwkv_engine::load_place(int id, const StFile& f, float alpha) {
    CK(cudaSetDevice(dev));
    __half* cols = reinterpret_cast<__half*>(ad_stage);
    uint4* blocks = reinterpret_cast<uint4*>(ad_stage + ad_stage_cols);
    for (const AdMatrix& m : ad_mats) {
        const StTensor* la = f.find(m.name + ".lora.0");
        if (!la) continue;
        const StTensor* lb = f.find(m.name + ".lora.1");
        const int r = (int)la->shape[1];
        const __half* b = reinterpret_cast<const __half*>(lb->data);
        std::vector<__half> e((size_t)m.N * GEMM_BK, __float2half_rn(0.f));
        for (int n = 0; n < m.N; ++n)
            for (int j = 0; j < r; ++j) e[(size_t)n * GEMM_BK + j] = __float2half_rn(alpha * __half2float(b[(size_t)n * r + j]));
        CK(cudaMemcpyAsync(cols, e.data(), e.size() * 2, cudaMemcpyHostToDevice, stream));
        launch_repack(num_sms, cols, GEMM_BK, 0, 0, m.N, GEMM_BK, blocks, stream);
        CK(cudaMemcpy2DAsync(m.W + (size_t)(m.kbw + id - 1) * GEMM_WBYTES, (size_t)m.KB * GEMM_WBYTES, blocks, GEMM_WBYTES,
                             GEMM_WBYTES, m.tiles, cudaMemcpyDeviceToDevice, stream));
        const std::vector<uint16_t> rows = adapter_a_rows(la->data, m.K, r);
        CK(cudaMemcpyAsync(m.A[id - 1], rows.data(), rows.size() * 2, cudaMemcpyHostToDevice, stream));
        set_place_rank(m, id, r);
    }
    CK(cudaStreamSynchronize(stream));
    place_full[id - 1] = 1;
    drop_adapter_graphs();
}

// b200rwkv_unload_adapter after its checks: zeros over place `id`'s tail block of every planned matrix, and rank 0 (the shrink
// then writes zeros into that tail block of the operand and reads none of the place's A rows).
void b200rwkv_engine::unload_place(int id) {
    CK(cudaSetDevice(dev));
    for (const AdMatrix& m : ad_mats) {
        CK(cudaMemset2DAsync(m.W + (size_t)(m.kbw + id - 1) * GEMM_WBYTES, (size_t)m.KB * GEMM_WBYTES, 0, GEMM_WBYTES, m.tiles,
                             stream));
        set_place_rank(m, id, 0);
    }
    CK(cudaStreamSynchronize(stream));
    place_full[id - 1] = 0;
    drop_adapter_graphs();
}

// the shrink launch of one step phase: (8 columns, 16 rows, projection) CTAs over the step's token rows, or its output rows
void b200rwkv_engine::enqueue_shrink(const AdapterParams& p0, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    if (p0.nproj == 0) return;
    AdapterParams p = p0;
    p.th = p.head ? sh.th_rows : sh.th;
    const dim3 grid = adapter_grid(p.head ? 16 * sh.MTR : sh.rows, p.nproj);
    if (sh.split) launch_k(adapter_shrink_kernel<true>, grid, dim3(AD_THREADS), 0, p, KC_OTHER, s, prof);
    else launch_k(adapter_shrink_kernel<false>, grid, dim3(AD_THREADS), 0, p, KC_OTHER, s, prof);
}

// -----------------------------------------------------------------------------------------
// one forward step over the tokens described by d_meta
// -----------------------------------------------------------------------------------------
void b200rwkv_engine::enqueue_step(cudaStream_t s, const StepShape& sh, Profiler* prof) {
    launches_last_step = 0;
    last_sh = sh;
    auto gemm = [&](const GemmLaunch& g, bool head = false) {
        GemmLaunch g2 = g;
        if (d_step_trace && trace_capture) {
            g2.p.trace = tr_next(1000000 + (int)(g.weight_bytes >> 20));
            if ((long long)step_trace_bytes.size() <= launches_last_step) step_trace_bytes.resize(launches_last_step + 1, 0);
            step_trace_bytes[launches_last_step] = (long long)g.weight_bytes;
        }
        if (prof) prof->weight_bytes += g.weight_bytes;
        launch_gemm(g2, sh, s, prof, head);
    };
    launch_embed(embed, sh, s, prof);
    // snapshot steps: offsets of one layer's parts in a snapshot record [L][C | Hl*N*N | C]
    const size_t W = (size_t)Hl * N * N, rec = 2 * (size_t)C + W;
    float* const* snap_rec = sh.snap ? snap_rec_dev() : nullptr;
    auto ln_stage = [&](const LnMixParams& lp0, size_t snap_off) {
        LnMixParams lp = lp0;
        lp.trace = tr_next(0);
        lp.snap_rec = snap_rec; lp.snap_off = snap_off;
        launch_ln(lp, sh, s, prof);
    };
    for (int l = 0; l < L; ++l) {
        Layer& ly = layers[l];
        AdLayer* ad = sh.ad ? &ad_layers[l] : nullptr;      // a slot of the step is bound: W' plans and their shrinks
        // LN1 of layer l commits the channel-mix shift of layer l - 1 (layer 0's commits nothing), LN2 the time-mix shift
        const size_t off_ffn_prev = l > 0 ? (size_t)(l - 1) * rec + C + W : 0, off_att = (size_t)l * rec;
        if (ly.has_pre6 && (sh.MT == 1 || batch_inv)) {
            // batch-invariant steps of > 16 tokens: LN1 as its own wide cluster launch, then the front half's phases 2 and 3
            if (sh.MT > 1) ln_stage(ly.ln1, off_ffn_prev);
            Pre6Params q = ly.pre6;
            q.ln = ly.ln1;
            q.ln.trace = tr_next(6);
            q.ln.snap_rec = snap_rec; q.ln.snap_off = off_ffn_prev;
            launch_pre6(q, sh, s, prof);
        } else {
            ln_stage(ly.ln1, off_ffn_prev);
            for (auto& g : ly.lora) gemm(g);
        }
        if (ad) enqueue_shrink(ad->s_pre, sh, s, prof);
        for (auto& g : ad ? ad->pre : ly.pre) gemm(g);
        {
            WkvParams wp = ly.wkv;
            wp.trace = tr_next(2);
            wp.snap_rec = snap_rec; wp.snap_off = off_att + C;
            launch_wkv(wp, sh, s, prof);
        }
        if (ad) enqueue_shrink(ad->s_o, sh, s, prof);
        gemm(ad ? ad->o : ly.o);
        if (world > 1) launch_k(tp_barrier_kernel, dim3(1), dim3(32), 0, tpbar, KC_OTHER, s, prof);
        ln_stage(ly.ln2, off_att);
        if (ad) {
            enqueue_shrink(ad->s_fk, sh, s, prof);
            gemm(ad->ffn[0]);
            enqueue_shrink(ad->s_fv, sh, s, prof);
            gemm(ad->ffn[1]);
        } else {
            for (auto& g : ly.ffn) gemm(g);
        }
        if (world > 1) launch_k(tp_barrier_kernel, dim3(1), dim3(32), 0, tpbar, KC_OTHER, s, prof);
    }
    {
        LnOutParams lo = lnout;
        if (sh.snap) {
            lo.snap_rec = snap_rec; lo.snap_off = (size_t)(L - 1) * rec + C + W;
            if (sh.MTX > 0) {
                lo.snap_meta = MetaView{reinterpret_cast<const int*>(snap_dev.p), maxT, S};
                lo.snap_head_in = a_snap_head.p;
            }
        }
        launch_ln_out(lo, sh, s, prof);
    }
    // a quantised head (b200rwkv_head_format) has no W' plan, so its bound steps' shrink launches are empty
    if (sh.MTR > 0 && sh.ad) {
        enqueue_shrink(s_head, sh, s, prof);
        gemm(head_plan(true), true);
    } else if (sh.MTR > 0) {
        gemm(head_plan(false), true);
    }
    if (sh.MTX > 0) {        // the snapshot tokens without an output row: a head launch of their own, the main one unchanged
        StepShape shx = sh;
        shx.MTR = sh.MTX;
        shx.th_rows = sh.split ? 32 : 16 * sh.MTX;
        if (sh.ad) enqueue_shrink(s_snap_head, shx, s, prof);
        if (prof) prof->weight_bytes += head_plan(false).weight_bytes;
        launch_gemm(snap_head_plan(sh.ad), shx, s, prof, true);
    }
    if (world > 1) launch_k(tp_barrier_kernel, dim3(1), dim3(32), 0, tpbar, KC_OTHER, s, prof);
}

// embedding gather + LN0 of a step: one CTA per token row, CTAs past T exit
LnPick b200rwkv_engine::launch_embed(const EmbedParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    launch_k(embed_ln0_kernel, dim3(sh.rows), dim3(LN_THREADS), 0, p, KC_LN, s, prof);
    return {LNK_EMBED, ln_nv(p.C), 0};
}

// LN1 / LN2 of a step: the 16 x 8 cluster kernel when the whole step is decode-shaped and the row fits its slices (split
// operands with precision 1), else one CTA per token row.  In the batch-invariant mode a longer step runs the cluster
// kernel's WIDE variant, one cluster per token row.
LnPick b200rwkv_engine::launch_ln(const LnMixParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    LnMixParams lp = p;
    lp.kq_tile = sh.th;
    if (ln_cluster_ok && sh.MT > 1 && batch_inv) {
        launch_cluster = PRE_CLUSTER;
        launch_k(ln_mix_cluster_kernel<false, true>, dim3(PRE_CLUSTER * sh.rows), dim3(PRE_THREADS), 0, lp, KC_LN, s, prof);
        return {LNK_MIX_CLUSTER_WIDE, 1, 0};
    }
    if (ln_cluster_ok && sh.MT == 1) {
        launch_cluster = PRE_CLUSTER;
        if (sh.split) launch_k(ln_mix_cluster_kernel<true>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, lp, KC_LN, s, prof);
        else launch_k(ln_mix_cluster_kernel<false>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, lp, KC_LN, s, prof);
        return {LNK_MIX_CLUSTER, 1, sh.split ? 1 : 0};
    }
    launch_k(ln_mix_kernel, dim3(sh.rows), dim3(LN_THREADS), 0, lp, KC_LN, s, prof);
    return {LNK_MIX, ln_nv(p.C), 0};
}

// RWKV-6 decode front half (LN1 + token shift + ddlerp LoRA) as one launch of 16 clusters x 8; the caller checked
// pre6_fits(q.Dm, C) and that the step is decode-shaped (MT == 1), or, in the batch-invariant mode, launched LN1 of the
// longer step before it (the WIDE variant runs phases 2 and 3 over its token groups)
LnPick b200rwkv_engine::launch_pre6(const Pre6Params& q0, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    Pre6Params q = q0;
    q.ln.kq_tile = sh.th;
    launch_cluster = PRE_CLUSTER;
    if (sh.MT > 1) {
        if (q.Dm == 32) launch_k(pre6_kernel<2, false, true>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
        else launch_k(pre6_kernel<4, false, true>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
        return {LNK_PRE6_WIDE, q.Dm / 16, 0};
    }
    if (sh.split) {
        if (q.Dm == 32) launch_k(pre6_kernel<2, true>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
        else launch_k(pre6_kernel<4, true>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
    } else {
        if (q.Dm == 32) launch_k(pre6_kernel<2, false>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
        else launch_k(pre6_kernel<4, false>, dim3(PRE_GRID), dim3(PRE_THREADS), 0, q, KC_LN, s, prof);
    }
    return {LNK_PRE6, q.Dm / 16, sh.split ? 1 : 0};
}

// final residual update + ln_out of a step into the head operand, which holds the step's output rows (and, on a snapshot
// step, into the snapshot rows' head operand of sh.MTX token tiles)
LnPick b200rwkv_engine::launch_ln_out(const LnOutParams& p, const StepShape& sh, cudaStream_t s, Profiler* prof) {
    LnOutParams lo = p;
    lo.kq_tile = sh.th_rows;
    if (lo.snap_head_in) lo.snap_kq = sh.split ? 32 : 16 * sh.MTX;
    if (sh.split) launch_k(ln_out_kernel<true>, dim3(sh.rows), dim3(LN_THREADS), 0, lo, KC_LN, s, prof);
    else launch_k(ln_out_kernel<false>, dim3(sh.rows), dim3(LN_THREADS), 0, lo, KC_LN, s, prof);
    return {LNK_OUT, ln_nv(p.C), sh.split ? 1 : 0};
}

static inline int mt_bucket(int rows) { return rows <= 16 ? 1 : (rows <= 32 ? 2 : (rows <= 64 ? 4 : 8)); }

// The shape of a step of T tokens and R output rows, for every launch of it.  Split operands only when the whole step is
// decode-shaped: a precision-1 engine keeps its steps at <= 16 tokens (infer), the head's operand then holds 32 rows too.
StepShape b200rwkv_engine::step_shape(int T, int R) const {
    StepShape sh;
    sh.MT = mt_bucket(T);
    sh.MTR = R > 0 ? mt_bucket(R) : 0;
    sh.rows = 16 * sh.MT;
    sh.split = split_on && sh.MT == 1;
    sh.th = sh.split ? 32 : sh.rows;
    sh.th_rows = sh.split ? 32 : 16 * sh.MTR;
    return sh;
}

// last logits row of every slot of this step -> keep[slot] (rank 0 gathers the vocabulary shards); see sample.cuh
void b200rwkv_engine::enqueue_keep(cudaStream_t s, int MTR) {
    if (MTR <= 0 || rank != 0 || !d_keep) return;
    KeepParams kp;
    memset(&kp, 0, sizeof(kp));
    for (int q = 0; q < world; ++q) kp.shard[q] = (const float*)(peer_base[q] + off_logits);
    kp.world = world; kp.Vl = Vl; kp.V = V;
    kp.meta = MetaView{d_meta, maxT, S};
    kp.keep = d_keep;
    launch_k(keep_rows_kernel, dim3(MTR * 16, KEEP_CHUNKS), dim3(KEEP_THREADS), 0, kp, KC_OTHER, s, nullptr);
}

// the logits row of every snapshot token of this step -> its snapshot (the tables b200rwkv_engine::infer uploaded)
void b200rwkv_engine::enqueue_snap_rows(cudaStream_t s, const StepShape& sh) {
    SnapRowParams sp;
    sp.src = reinterpret_cast<const float* const*>(snap_rec_dev() + maxT);
    sp.dst = snap_rec_dev() + 2 * maxT;
    sp.V = V;
    launch_k(snap_rows_kernel, dim3(sh.rows, KEEP_CHUNKS), dim3(KEEP_THREADS), 0, sp, KC_OTHER, s, nullptr);
}

void b200rwkv_engine::run_step(const StepShape& sh) {
    const int key = sh.MT * 8 + sh.MTR + (sh.ad ? 128 : 0) + (sh.snap ? 256 * (1 + sh.MTX) : 0);
    auto it = graphs.find(key);
    if (it == graphs.end()) {
        GraphExec ge = capture_graph(stream, [&] {
            enqueue_step(stream, sh, nullptr);
            enqueue_keep(stream, sh.MTR);
            if (sh.snap) enqueue_snap_rows(stream, sh);
        });
        it = graphs.emplace(key, StepGraph{std::move(ge), launches_last_step}).first;
    }
    CK(cudaGraphLaunch(it->second.exec, stream));
    launch_total += it->second.launches;         // kernels of THIS graph, not of whichever was captured last
    last_sh = sh;                                // a replay of a cached graph runs this shape, whatever was captured last
}

// The device table of step buffers the LN stages record into: cell l is set for the layers keep_hidden_layers or
// keep_hidden_pooled asked for (layer L - 1 comes from ln_out_kernel's d_hidden and has no cell).  A layer both asked for
// is recorded once, into the kept layer's buffer.
void b200rwkv_engine::upload_hid_tab() {
    std::vector<float*> tab(L, nullptr);
    for (size_t k = 0; k < hid_layers.size(); ++k)
        if (hid_layers[k] < L - 1) tab[hid_layers[k]] = hid_step + k * maxT * C;
    for (size_t k = 0; k < pool_layers.size(); ++k) {
        const int l = pool_layers[k];
        if (l < L - 1 && !tab[l]) tab[l] = pool_step + k * maxT * C;
        pool_src[k] = l == L - 1 ? d_hidden : tab[l];
    }
    // on the engine's stream and complete before returning: the step kernels read the table before griddepcontrol.wait
    CK(cudaMemcpyAsync(d_hid_tab, tab.data(), tab.size() * sizeof(float*), cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
}

// The snapshot step block and the snapshot rows' head launches (b200rwkv_infer_snapshots), made on first use: the copies of
// head / ad_head read a_snap_head and write snap_logits, over the snapshot metadata's R rows, with counters of their own.
void b200rwkv_engine::snap_setup() {
    if (snap_dev) return;
    snap_sizes();
    snap_dev = Buf<uint8_t>(snap_bytes);
    snap_host = HostBuf<uint8_t>(snap_bytes * META_RING);
    const int K = n_adapters ? (cdiv(C, GEMM_BK) + n_adapters) * GEMM_BK : C;      // a_head's columns
    a_snap_head = a16_alloc(K);
    snap_logits = Buf<float>((size_t)maxT * V * 4);
    const int* smeta = reinterpret_cast<const int*>(snap_dev.p);
    snap_head = snap_rebase(head, (unsigned*)dalloc((size_t)head.total_tiles * 4, true));
    if (n_adapters) {
        snap_ad_head = snap_rebase(ad_head, (unsigned*)dalloc((size_t)ad_head.total_tiles * 4, true));
        s_snap_head = s_head;
        s_snap_head.meta = MetaView{smeta, maxT, S};
        for (int k = 0; k < s_snap_head.nproj; ++k) s_snap_head.p[k].op = a_snap_head.p + (s_head.p[k].op - a_head.p);
    }
    if (qhead.plan.qtype != QT_NONE) qhead.snap = snap_rebase(qhead.plan, qhead.snap_counters);
}

// A head launch over the snapshot rows: a_snap_head into snap_logits, over the snapshot metadata's R rows, with `counters`
// (zeroed, total_tiles of them) of its own
GemmLaunch b200rwkv_engine::snap_rebase(const GemmLaunch& g, unsigned* counters) const {
    GemmLaunch x = g;
    for (int i = 0; i < x.p.nseg; ++i) {
        x.p.seg[i].A = a_snap_head.p + (x.p.seg[i].A - a_head.p);
        x.p.seg[i].out = snap_logits.p + ((float*)x.p.seg[i].out - d_logits);
    }
    x.p.nrows = reinterpret_cast<const int*>(snap_dev.p) + 2;
    x.p.counters = counters;
    return x;
}

// b200rwkv_head_format after its checks: the codes of head.weight in format `qt` (QT_NONE: none), quantised from the f16 head's
// own blocks, unpacked into dense rows; the fill that derives them again on a weight update; the plans over them.  Everything
// is allocated and written before the engine changes, so a failure leaves the previous head in place.  The captured step
// graphs hold the old head launch and are dropped.
void b200rwkv_engine::set_head_format(int qt) {
    CK(cudaSetDevice(dev));
    QHead q;
    Fill f;
    if (qt != QT_NONE) {
        const int tiles = head.total_tiles, KB = head.p.seg[0].KB;       // one segment: [V][C], C a multiple of 128
        const size_t code_bytes = (size_t)tiles * KB * q_block_bytes(qt);
        q.codes = Buf<uint8_t>(code_bytes + (qt == QT_FP8 ? (size_t)tiles * FP8_SCALE_BYTES : 0));
        q.counters = Buf<unsigned>((size_t)tiles * 4);
        q.snap_counters = Buf<unsigned>((size_t)tiles * 4);
        Buf<__half> rows((size_t)V * C * 2);
        CK(cudaMemsetAsync(q.counters, 0, q.counters.bytes, stream));
        CK(cudaMemsetAsync(q.snap_counters, 0, q.snap_counters.bytes, stream));
        const size_t nchunk = (size_t)tiles * KB * (GEMM_WBYTES / 16);
        const int grid = (int)std::min<size_t>((nchunk + 255) / 256, (size_t)num_sms * 16);
        unpack_weight_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint4*>(head.p.W), V, C, tiles, KB, rows);
        CK(cudaGetLastError());
        f.kind = FILL_SEG; f.ld = C; f.N = V; f.K = C; f.tiles = tiles; f.kb = KB; f.qtype = qt; f.dst = q.codes.p;
        f.plan = B200RWKV_PLAN_HEAD;
        if (qt == QT_FP8) f.scales = reinterpret_cast<float*>(q.codes.p + code_bytes);
        run_fill(f, rows, stream);
        CK(cudaStreamSynchronize(stream));
        gemm_smem_limits(qt);
        q.plan = head;
        q.plan.qtype = qt;
        q.plan.weight_bytes = quant_matrix_bytes(qt, V, C);
        q.plan.p.W = q.codes;
        q.plan.p.scales = f.scales;
        q.plan.p.counters = q.counters;
        if (snap_dev) q.snap = snap_rebase(q.plan, q.snap_counters);
    }
    std::vector<Fill>& hf = fills.at("head.weight");
    if (qhead.plan.qtype != QT_NONE) hf.pop_back();       // the previous format's fill, pushed last
    if (qt != QT_NONE) hf.push_back(f);
    graphs.clear();
    qhead = std::move(q);        // q now holds the previous codes, released on return (cudaFree waits for the device)
}

// allocate a snapshot record (+ a logits row when this rank keeps them)
static Snapshot snapshot_alloc(b200rwkv_engine* e, bool with_logits) {
    Snapshot sn;
    const size_t rec = 2 * (size_t)e->C + (size_t)e->Hl * e->N * e->N;
    sn.buf = Buf<float>(rec * e->L * 4);
    if (with_logits) sn.logits = Buf<float>((size_t)e->V * 4);
    return sn;
}

// fills one step's metadata; returns T
int b200rwkv_engine::fill_meta(int* m, const std::vector<int>& slots, const std::vector<int>& counts,
                               const std::vector<const uint32_t*>& toks, const std::vector<int>& outmode, int* R_out) {
    MetaView mv{m, maxT, S};
    int* tok = const_cast<int*>(mv.tok());
    int* tslot = const_cast<int*>(mv.tok_slot());
    int* tprev = const_cast<int*>(mv.tok_prev());
    int* tlast = const_cast<int*>(mv.tok_last());
    int* otok = const_cast<int*>(mv.out_tok());
    int* torow = const_cast<int*>(mv.tok_outrow());
    int* sid = const_cast<int*>(mv.slot_id());
    int* sstart = const_cast<int*>(mv.slot_start());
    int* scount = const_cast<int*>(mv.slot_count());
    int T = 0, R = 0;
    for (size_t i = 0; i < slots.size(); ++i) {
        sid[i] = slots[i];
        sstart[i] = T;
        scount[i] = counts[i];
        for (int j = 0; j < counts[i]; ++j, ++T) {
            tok[T] = (int)toks[i][j];
            tslot[T] = slots[i];
            tprev[T] = (j == 0) ? -1 : T - 1;
            tlast[T] = (j == counts[i] - 1) ? 1 : 0;
            const bool out = (outmode[i] == 2) || (outmode[i] == 1 && j == counts[i] - 1);
            torow[T] = out ? R : -1;
            if (out) otok[R++] = T;
        }
    }
    m[0] = T; m[1] = (int)slots.size(); m[2] = R;
    *R_out = R;
    return T;
}

// Fills one snapshot step block hs [snap_bytes] from the step's metadata hm (T tokens) and its snapshot tokens: the record of
// each token row, where its logits row comes from and goes to, and a copy of the metadata whose output rows are the
// snapshot tokens without one, in the order of `tk`.  Returns X, the number of those rows.
int b200rwkv_engine::fill_snap(uint8_t* hs, const int* hm, int T, const std::vector<SnapTok>& tk) const {
    int* smeta = reinterpret_cast<int*>(hs);
    float** rec = reinterpret_cast<float**>(hs + snap_meta_bytes);
    const float** src = const_cast<const float**>(rec + maxT);
    float** dst = rec + 2 * maxT;
    memset(hs + snap_meta_bytes, 0, 3 * (size_t)maxT * sizeof(void*));
    memcpy(smeta, hm, meta_ints * 4);
    MetaView sv{smeta, maxT, S};
    int* s_outrow = const_cast<int*>(sv.tok_outrow());
    int* s_outtok = const_cast<int*>(sv.out_tok());
    const int* torow = MetaView{hm, maxT, S}.tok_outrow();
    for (int t = 0; t < T; ++t) s_outrow[t] = -1;
    int X = 0;
    for (const SnapTok& a : tk) {
        const int t = a.t;
        rec[t] = a.rec;
        dst[t] = a.row;
        if (torow[t] >= 0) {
            src[t] = d_logits + (size_t)torow[t] * V;
        } else {
            s_outrow[t] = X;
            s_outtok[X] = t;
            src[t] = snap_logits + (size_t)X * V;
            ++X;
        }
    }
    smeta[2] = X;
    return X;
}

void b200rwkv_engine::infer(int nslot, const int32_t* slot, const int32_t* ntok, const uint32_t* tokens, const int32_t* option,
                            float* logits_out, size_t cap, int32_t* rows_out, const ScoreOut* score, const SnapPlan* snap) {
    REQUIRE(nslot >= 0 && (nslot == 0 || (slot && ntok && option)), B200RWKV_ERR_INVALID, "infer: null argument");
    REQUIRE(connected, B200RWKV_ERR_INVALID, "tensor-parallel engine is not connected (b200rwkv_tp_connect)");
    const int max_option = score ? B200RWKV_OPTION_SCORE : B200RWKV_OPTION_NONE;
    std::vector<char> seen(S, 0);
    size_t total_rows = 0, total_tok = 0, total_score = 0;
    for (int i = 0; i < nslot; ++i) {
        REQUIRE(slot[i] >= 0 && slot[i] < S, B200RWKV_ERR_STATE, "infer: slot out of range");
        REQUIRE(!seen[slot[i]], B200RWKV_ERR_INVALID, "infer: duplicate slot in one call");
        seen[slot[i]] = 1;
        REQUIRE(ntok[i] >= 0, B200RWKV_ERR_INVALID, "infer: negative token count");
        REQUIRE(option[i] >= B200RWKV_OPTION_LAST && option[i] <= max_option, B200RWKV_ERR_INVALID, "infer: bad option");
        const int r = (option[i] == B200RWKV_OPTION_FULL) ? ntok[i] : ((option[i] == B200RWKV_OPTION_LAST && ntok[i] > 0) ? 1 : 0);
        if (rows_out) rows_out[i] = r;
        total_rows += (size_t)r;
        total_tok += (size_t)ntok[i];
        if (option[i] == B200RWKV_OPTION_SCORE) total_score += (size_t)ntok[i];
    }
    const bool any_score = score && std::any_of(option, option + nslot, [](int32_t o) { return o == B200RWKV_OPTION_SCORE; });
    REQUIRE(!any_score || score->score, B200RWKV_ERR_INVALID, "infer_ex: score_out is NULL but the call has SCORE entries");
    REQUIRE(!any_score || world == 1, B200RWKV_ERR_UNSUPPORTED, "infer_ex: OPTION_SCORE is not supported under tensor parallelism");
    REQUIRE(total_tok == 0 || tokens, B200RWKV_ERR_INVALID, "infer: null tokens");
    for (size_t i = 0; i < total_tok; ++i)
        REQUIRE(tokens[i] < (uint32_t)V, B200RWKV_ERR_INVALID, "infer: token id " + std::to_string(tokens[i]) + " is outside the vocabulary");
    const bool want_logits = (rank == 0);          // tensor parallel: rank 0 gathers all vocabulary shards
    REQUIRE(!want_logits || !logits_out || total_rows * (size_t)V <= cap || total_rows == 0, B200RWKV_ERR_INVALID, "infer: logits buffer too small");
    // snapshots: every check before any CUDA call, then the records (new ones, or reused ids overwritten in place)
    const int nsnap = snap ? snap->n : 0;
    // records of ids 0, and rows for reused ids that had none: entered into `snaps` only once the call has run, so a failed
    // call leaves no id with a row it never wrote
    std::vector<Snapshot> snap_new;
    std::vector<std::pair<uint64_t, Buf<float>>> row_new;
    struct SnapDst { int tok; float* state; float* row; };
    std::vector<std::vector<SnapDst>> snap_at(nslot);      // per entry: token index, record, logits row
    if (snap) {
        REQUIRE(nsnap >= 0, B200RWKV_ERR_INVALID, "infer_snapshots: negative snapshot count");
        REQUIRE(nsnap == 0 || (snap->entry && snap->tok && snap->ids), B200RWKV_ERR_INVALID, "infer_snapshots: null argument");
        REQUIRE(nsnap == 0 || world == 1, B200RWKV_ERR_UNSUPPORTED, "infer_snapshots: snapshots are not supported under tensor parallelism");
        std::set<std::pair<int, int>> at;
        std::set<uint64_t> reused;
        for (int k = 0; k < nsnap; ++k) {
            const int i = snap->entry[k], p = snap->tok[k];
            REQUIRE(i >= 0 && i < nslot, B200RWKV_ERR_INVALID, "infer_snapshots: entry index out of range");
            REQUIRE(p >= 1 && p <= ntok[i], B200RWKV_ERR_INVALID, "infer_snapshots: position outside [1, ntok] of its entry");
            REQUIRE(at.insert({i, p}).second, B200RWKV_ERR_INVALID, "infer_snapshots: duplicate (entry, position)");
            const uint64_t id = snap->ids[k];
            if (id == 0) continue;
            REQUIRE(reused.insert(id).second, B200RWKV_ERR_INVALID, "infer_snapshots: snapshot id listed twice");
            REQUIRE(snaps.count(id), B200RWKV_ERR_STATE, "infer_snapshots: unknown snapshot id");
        }
    }
    if (nsnap > 0) {
        snap_setup();
        for (int k = 0; k < nsnap; ++k) {
            float *state, *row;
            if (snap->ids[k] == 0) {
                snap_new.push_back(snapshot_alloc(this, true));
                state = snap_new.back().buf;
                row = snap_new.back().logits;
            } else {
                Snapshot& sn = snaps.at(snap->ids[k]);
                state = sn.buf;
                row = sn.logits;
                if (!row) {
                    row_new.emplace_back(snap->ids[k], Buf<float>((size_t)V * 4));
                    row = row_new.back().second;
                }
            }
            snap_at[snap->entry[k]].push_back({snap->tok[k] - 1, state, row});
        }
    }
    // logits_out == NULL: the rows stay in HBM (b200rwkv_sample_topk reads the last row of every slot from there)
    const bool copy_logits = want_logits && logits_out != nullptr;
    // f32-activation mode runs every step decode-shaped (<= 16 tokens): the split-operand kernels are the 16-token ones
    const int step_cap = std::min(chunk, split_on ? 16 : maxT);
    // Step packing: every step shares its token budget evenly over the entries that still have tokens (web-rwkv shares the
    // chunk "fairly across slots", SURVEY.md A4; results do not depend on the cut).  Many slots with one token each keep
    // the WKV kernels wide (one CTA per head and slot) where a single slot with 64 tokens would run them 40 CTAs wide.
    std::vector<size_t> base(nslot + 1, 0), row_base(nslot + 1, 0);
    std::vector<int> pos(nslot, 0), rows_done(nslot, 0);
    for (int i = 0; i < nslot; ++i) {
        base[i + 1] = base[i] + (size_t)ntok[i];
        const int r = (option[i] == B200RWKV_OPTION_FULL) ? ntok[i] : ((option[i] == B200RWKV_OPTION_LAST && ntok[i] > 0) ? 1 : 0);
        row_base[i + 1] = row_base[i] + (size_t)r;
    }
    // SCORE entries: score index of token j of entry i is score_base[i] + j.  Token 0 is scored from the slot's kept row,
    // token j >= 1 from the row the step produced after token j - 1 (the entry's last row gets no target).  Each scoring
    // launch reads its own slice of the pinned row list (never rewritten within the call).
    std::vector<size_t> score_base(nslot + 1, 0);
    for (int i = 0; i < nslot; ++i) score_base[i + 1] = score_base[i] + (option[i] == B200RWKV_OPTION_SCORE ? (size_t)ntok[i] : 0);
    ScoreRow* sc_rows = nullptr;
    size_t sc_used = 0;
    // b200rwkv_score_top: n best entries of each scored row, after the score fields of sc_dev / sc_host
    const int tn = top_n;
    const size_t top_bytes = (size_t)tn * 8;         // per scored token: tn ids, tn logprobs
    auto launch_score = [&](size_t first, size_t n) {
        if (n == 0) return;
        ScoreParams sp;
        sp.rows = reinterpret_cast<const ScoreRow*>(sc_dev.p) + first;
        sp.V = V;
        sp.score = reinterpret_cast<float*>(sc_dev + total_score * sizeof(ScoreRow));
        sp.argmax = reinterpret_cast<unsigned*>(sc_dev + total_score * (sizeof(ScoreRow) + 4));
        CK(cudaMemcpyAsync(sc_dev + first * sizeof(ScoreRow), sc_rows + first, n * sizeof(ScoreRow), cudaMemcpyHostToDevice, stream));
        score_rows_kernel<<<(unsigned)n, SCORE_THREADS, 0, stream>>>(sp);
        CK(cudaGetLastError());
        if (tn > 0) {
            ScoreTopParams tp;
            tp.rows = sp.rows;
            tp.V = V;
            tp.nseg = cdiv(V, TOPK_SEG);
            tp.top_n = tn;
            tp.cand_x = top_cand_x;
            tp.cand_id = top_cand_id;
            tp.out_id = reinterpret_cast<unsigned*>(sc_dev + total_score * (sizeof(ScoreRow) + 8));
            tp.out_lp = reinterpret_cast<float*>(sc_dev + total_score * (sizeof(ScoreRow) + 8) + total_score * tn * 4);
            score_top_segment_kernel<<<dim3(tp.nseg, (unsigned)n), TOPK_SEG_THREADS, 0, stream>>>(tp);
            CK(cudaGetLastError());
            score_top_merge_kernel<<<(unsigned)n, TOPK_MERGE_THREADS, 0, stream>>>(tp);
            CK(cudaGetLastError());
        }
    };
    top_last_n = 0;
    top_last_rows = 0;
    if (total_score > 0) {
        const size_t row_bytes = sizeof(ScoreRow) + 8 + top_bytes;
        const size_t want = total_score * row_bytes, bytes = std::max<size_t>(want, 256 * row_bytes);
        sc_dev.grow(want, bytes);
        sc_host.grow(want, bytes);
        sc_rows = reinterpret_cast<ScoreRow*>(sc_host.p);
        std::lock_guard<std::mutex> lk(keep_mu);
        for (int i = 0; i < nslot; ++i)
            if (option[i] == B200RWKV_OPTION_SCORE && ntok[i] > 0)
                sc_rows[sc_used++] = {keep_valid[slot[i]] ? d_keep + (size_t)slot[i] * V : nullptr, tokens[base[i]], (unsigned)score_base[i]};
    }
    launch_score(0, sc_used);          // before the first step replaces the kept rows
    {       // a NONE entry with tokens moves its slot's state past the kept row and writes no new one
        std::lock_guard<std::mutex> lk(keep_mu);
        for (int i = 0; i < nslot; ++i)
            if (option[i] == B200RWKV_OPTION_NONE && ntok[i] > 0) keep_valid[slot[i]] = 0;
    }
    if (hidden_keep) d_hidden_all.grow(total_tok * C * 4, std::max<size_t>(total_tok, 256) * C * 4);
    hidden_rows = 0;
    const size_t n_hid = hid_layers.size();
    hid_last.clear();
    hid_last_rows = 0;
    hid_all.grow(n_hid * total_tok * C * 4, n_hid * std::max<size_t>(total_tok, 256) * C * 4);
    // pooled rows: every step lists its entries in its own slice of the pinned list (never rewritten within the call); an
    // entry takes at least one token of every step it is in, so the call's tokens bound the list
    const size_t n_pool = pool_layers.size();
    pool_last.clear();
    size_t pool_used = 0;
    if (n_pool) {
        const size_t bytes = std::max<size_t>(total_tok, 256) * sizeof(PoolEntry);
        pool_dev.grow(total_tok * sizeof(PoolEntry), bytes);
        pool_host.grow(total_tok * sizeof(PoolEntry), bytes);
    }
    int step_no = 0;
    for (;;) {
        int n_active = 0;
        for (int i = 0; i < nslot; ++i) n_active += (pos[i] < ntok[i]);
        if (n_active == 0) break;
        std::vector<int> s_entry, s_slots, s_counts, s_out;
        std::vector<const uint32_t*> s_toks;
        // at least WKV_STAGE_TOK tokens per slot and step while prompts are long: a WKV CTA then loads and stores its 16 KB
        // of state once per four tokens (staged path) and a step touches a quarter of the slots' states
        const int quota = std::max(WKV_STAGE_TOK, step_cap / n_active);
        int used = 0;
        for (int i = 0; i < nslot && used < step_cap; ++i) {
            const int remain = ntok[i] - pos[i];
            if (remain <= 0) continue;
            const int take = std::min({remain, quota, step_cap - used});
            s_entry.push_back(i);
            s_counts.push_back(take);
            used += take;
        }
        for (size_t j = 0; j < s_entry.size() && used < step_cap; ++j) {      // left-over budget, in entry order
            const int i = s_entry[j];
            const int extra = std::min(ntok[i] - pos[i] - s_counts[j], step_cap - used);
            s_counts[j] += extra;
            used += extra;
        }
        for (size_t j = 0; j < s_entry.size(); ++j) {
            const int i = s_entry[j];
            s_slots.push_back(slot[i]);
            s_toks.push_back(tokens + base[i] + pos[i]);
            const bool finishes = (pos[i] + s_counts[j] == ntok[i]);
            // SCORE runs the head exactly as FULL does (same step graph, same kept row): only where the rows go differs
            const bool all_rows = option[i] == B200RWKV_OPTION_FULL || option[i] == B200RWKV_OPTION_SCORE;
            s_out.push_back(all_rows ? 2 : ((finishes && option[i] == B200RWKV_OPTION_LAST) ? 1 : 0));
        }
        auto dev_rows = [&](size_t j) { return s_out[j] == 2 ? s_counts[j] : (s_out[j] == 1 ? 1 : 0); };
        auto scored = [&](size_t j) { return option[s_entry[j]] == B200RWKV_OPTION_SCORE; };
        // pinned metadata ring: a buffer is rewritten only after the copy that read it has completed
        const int mb = step_no % META_RING;
        if (step_no >= META_RING) CK(cudaEventSynchronize(meta_ev[mb]));
        int* hm = h_meta + (size_t)mb * meta_ints;
        int R = 0;
        const int T = fill_meta(hm, s_slots, s_counts, s_toks, s_out, &R);
        last_T = T;
        CK(cudaMemcpyAsync(d_meta, hm, meta_ints * 4, cudaMemcpyHostToDevice, stream));
        // snapshots of this step's tokens: their records, and where their logits rows come from
        int n_step_snap = 0, X = 0;
        if (nsnap > 0) {
            std::vector<SnapTok> tk;
            int t0 = 0;
            for (size_t j = 0; j < s_entry.size(); ++j) {
                const int i = s_entry[j];
                for (const SnapDst& a : snap_at[i])
                    if (a.tok >= pos[i] && a.tok < pos[i] + s_counts[j]) tk.push_back({t0 + (a.tok - pos[i]), a.state, a.row});
                t0 += s_counts[j];
            }
            n_step_snap = (int)tk.size();
            if (n_step_snap > 0) {
                uint8_t* hs = snap_host + (size_t)mb * snap_bytes;
                X = fill_snap(hs, hm, T, tk);
                CK(cudaMemcpyAsync(snap_dev, hs, snap_bytes, cudaMemcpyHostToDevice, stream));
            }
        }
        CK(cudaEventRecord(meta_ev[mb], stream));
        StepShape sh = step_shape(T, R);
        sh.ad = step_bound(s_slots);
        sh.snap = n_step_snap > 0;
        sh.MTX = X > 0 ? mt_bucket(X) : 0;
        run_step(sh);
        // step rows [T][C] -> the rows of every token of this call, in entry order
        auto gather_rows = [&](float* dst, const float* src) {
            int t0 = 0;
            for (size_t j = 0; j < s_entry.size(); ++j) {
                const int i = s_entry[j];
                CK(cudaMemcpyAsync(dst + (base[i] + pos[i]) * (size_t)C, src + (size_t)t0 * C, (size_t)s_counts[j] * C * 4,
                                   cudaMemcpyDeviceToDevice, stream));
                t0 += s_counts[j];
            }
        };
        if (hidden_keep) gather_rows(d_hidden_all, d_hidden);       // b200rwkv_last_hidden
        for (size_t k = 0; k < n_hid; ++k) gather_rows(hid_all + k * total_tok * C, hid_step_src((int)k));     // b200rwkv_last_hidden_layer
        if (n_pool) {        // b200rwkv_last_hidden_pooled: this step's rows into every entry's pooled row
            PoolEntry* pe = pool_host + pool_used;
            int t0 = 0;
            for (size_t j = 0; j < s_entry.size(); ++j) {
                const int i = s_entry[j];
                pe[j] = {t0, s_counts[j], i, pos[i], ntok[i]};
                t0 += s_counts[j];
            }
            CK(cudaMemcpyAsync(pool_dev + pool_used, pe, s_entry.size() * sizeof(PoolEntry), cudaMemcpyHostToDevice, stream));
            PoolParams pp;
            pp.ent = pool_dev + pool_used;
            std::copy(pool_src, pool_src + POOL_MAX_LAYERS, pp.src);
            pp.dst = pool_rows;
            pp.C = C; pp.dst_rows = S; pp.mode = pool_mode;
            hidden_pool_kernel<<<dim3((unsigned)s_entry.size(), (unsigned)n_pool, (unsigned)cdiv(C / 4, POOL_THREADS)), POOL_THREADS, 0,
                                 stream>>>(pp);
            CK(cudaGetLastError());
            ++launch_total;
            pool_used += s_entry.size();
        }
        if (sc_rows) {       // this step's SCORE rows, scored against each entry's next token
            const size_t first = sc_used;
            int r = 0;
            for (size_t j = 0; j < s_entry.size(); ++j) {
                const int i = s_entry[j];
                if (scored(j))
                    for (int t = 0; t < s_counts[j]; ++t) {
                        const int p = pos[i] + t;
                        if (p + 1 < ntok[i])
                            sc_rows[sc_used++] = {d_logits + (size_t)(r + t) * V, tokens[base[i] + p + 1], (unsigned)(score_base[i] + p + 1)};
                    }
                r += dev_rows(j);
            }
            launch_score(first, sc_used - first);
        }
        CK(cudaEventRecord(step_done, stream));
        if (R > 0) {
            std::lock_guard<std::mutex> lk(keep_mu);
            for (size_t i = 0; i < s_slots.size(); ++i)
                if (s_out[i] != 0) keep_valid[s_slots[i]] = 1;
        }
        if (R > 0 && copy_logits) {
            // rows of this step sit in entry order in d_logits; an entry's rows land at its own place of the entry-major
            // output, runs that are contiguous on both sides go out as one copy (SCORE rows stay on the device)
            int r0 = 0;
            size_t j = 0;
            while (j < s_entry.size()) {
                const int i = s_entry[j];
                int nr = dev_rows(j);
                if (nr == 0) { ++j; continue; }
                if (scored(j)) { r0 += nr; ++j; continue; }
                const size_t dst = row_base[i] + (size_t)rows_done[i];
                int run = nr;
                rows_done[i] += nr;
                size_t k = j + 1;
                while (k < s_entry.size()) {
                    const int i2 = s_entry[k];
                    const int nr2 = dev_rows(k);
                    if (nr2 == 0) { ++k; continue; }
                    if (scored(k)) break;
                    if (row_base[i2] + (size_t)rows_done[i2] != dst + (size_t)run) break;
                    rows_done[i2] += nr2;
                    run += nr2;
                    ++k;
                }
                float* o = logits_out + dst * (size_t)V;
                if (world == 1) {
                    CK(cudaMemcpyAsync(o, d_logits + (size_t)r0 * V, (size_t)run * V * 4, cudaMemcpyDeviceToHost, stream));
                } else {
                    for (int q = 0; q < world; ++q)      // column block q of every row, straight from rank q's shard
                        CK(cudaMemcpy2DAsync(o + (size_t)q * Vl, (size_t)V * 4, peer_base[q] + off_logits + (size_t)r0 * Vl * 4,
                                             (size_t)Vl * 4, (size_t)Vl * 4, run, cudaMemcpyDeviceToHost, stream));
                }
                r0 += run;
                j = k;
            }
        }      // (the next step's head projection is ordered after these copies by the stream)
        for (size_t j = 0; j < s_entry.size(); ++j) pos[s_entry[j]] += s_counts[j];
        ++step_no;
    }
    if (total_score > 0)      // scores, argmax ids and any top-n lists of the whole call: one copy
        CK(cudaMemcpyAsync(sc_host + total_score * sizeof(ScoreRow), sc_dev + total_score * sizeof(ScoreRow),
                           total_score * (8 + top_bytes), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    if (total_score > 0) {
        memcpy(score->score, sc_host + total_score * sizeof(ScoreRow), total_score * 4);
        if (score->argmax) memcpy(score->argmax, sc_host + total_score * (sizeof(ScoreRow) + 4), total_score * 4);
    }
    for (int k = 0, n = 0; k < nsnap; ++k)        // new snapshots get their ids once the call has run
        if (snap->ids[k] == 0) {
            const uint64_t id = next_snap++;
            snaps[id] = std::move(snap_new[n++]);
            snap->ids[k] = id;
        }
    for (auto& r : row_new) snaps.at(r.first).logits = std::move(r.second);
    if (hidden_keep) hidden_rows = (int)total_tok;
    hid_last = hid_layers;
    hid_last_rows = total_tok;
    pool_last = pool_layers;
    pool_last_ntok.assign(ntok, ntok + nslot);
    top_last_n = tn;
    top_last_rows = total_score;
}

// GPU sampling front half (sample.cuh).  Runs on the softmax stream under the softmax mutex: the reference samples from the
// task that owns softmax (run.rs:1237), concurrently with the infer task; the per-slot rows it reads are only rewritten by a
// step that contains the slot, which the host cannot submit before this call returned the slot's token.
// Argument checks of the sampling entries (sample_topk, sample_probs) that need no engine: the adjustment lists.
static void check_sample_lists(int nrows, const int32_t* pen_off, const uint32_t* pen_tok, const float* pen_val, const int32_t* bias_off,
                               const uint32_t* bias_tok, const float* bias_val, const char* who) {
    const std::string w(who);
    const int npen = pen_off ? pen_off[nrows] : 0, nbias = bias_off ? bias_off[nrows] : 0;
    REQUIRE(npen >= 0 && nbias >= 0 && (npen == 0 || (pen_tok && pen_val)) && (nbias == 0 || (bias_tok && bias_val)), B200RWKV_ERR_INVALID,
            w + ": bad adjustment lists");
    for (int i = 0; i < nrows; ++i) {
        REQUIRE(!pen_off || (pen_off[i] >= 0 && pen_off[i] <= pen_off[i + 1]), B200RWKV_ERR_INVALID, w + ": penalty offsets must ascend");
        REQUIRE(!bias_off || (bias_off[i] >= 0 && bias_off[i] <= bias_off[i + 1]), B200RWKV_ERR_INVALID, w + ": bias offsets must ascend");
    }
}

// The slot checks of the sampling entries: nrows in [1, max_batch], every slot in range, listed once, with a kept row.
void b200rwkv_engine::check_sample_slots(int nrows, const int32_t* slots, const char* who) {
    const std::string w(who);
    REQUIRE(nrows >= 1 && nrows <= S && slots, B200RWKV_ERR_INVALID, w + ": bad argument");
    std::lock_guard<std::mutex> lk(keep_mu);
    std::vector<char> seen(S, 0);
    for (int i = 0; i < nrows; ++i) {
        REQUIRE(slots[i] >= 0 && slots[i] < S, B200RWKV_ERR_STATE, w + ": slot out of range");
        REQUIRE(!seen[slots[i]], B200RWKV_ERR_INVALID, w + ": duplicate slot");
        seen[slots[i]] = 1;
        REQUIRE(keep_valid[slots[i]], B200RWKV_ERR_STATE, w + ": slot " + std::to_string(slots[i]) + " has produced no logits row yet");
    }
}

// Stages the slots and adjustment lists (checked) in one blob, uploads it on the softmax stream after the most recent step,
// and returns the device view.
SampleAdjust b200rwkv_engine::stage_sample_args(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok,
                                                const float* pen_val, const uint32_t* allow_bits, const int32_t* bias_off,
                                                const uint32_t* bias_tok, const float* bias_val) {
    const int npen = pen_off ? pen_off[nrows] : 0, nbias = bias_off ? bias_off[nrows] : 0;
    const size_t words = (size_t)(V + 31) / 32;
    auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
    // one staging blob: slot[n] | pen_off[n+1] | bias_off[n+1] | pen_tok | pen_val | bias_tok | bias_val | allow
    const size_t o_slot = 0, o_po = al(o_slot + (size_t)nrows * 4), o_bo = al(o_po + (size_t)(nrows + 1) * 4),
                 o_pt = al(o_bo + (size_t)(nrows + 1) * 4), o_pv = al(o_pt + (size_t)npen * 4), o_bt = al(o_pv + (size_t)npen * 4),
                 o_bv = al(o_bt + (size_t)nbias * 4), o_al = al(o_bv + (size_t)nbias * 4),
                 total = al(o_al + (allow_bits ? (size_t)nrows * words * 4 : 0));
    const size_t want = std::max<size_t>(total * 2, 1 << 20);
    tk_dev.grow(total, want);
    tk_host.grow(total, want);
    std::vector<int32_t> zeros(nrows + 1, 0);
    memcpy(tk_host + o_slot, slots, (size_t)nrows * 4);
    memcpy(tk_host + o_po, pen_off ? pen_off : zeros.data(), (size_t)(nrows + 1) * 4);
    memcpy(tk_host + o_bo, bias_off ? bias_off : zeros.data(), (size_t)(nrows + 1) * 4);
    if (npen) { memcpy(tk_host + o_pt, pen_tok, (size_t)npen * 4); memcpy(tk_host + o_pv, pen_val, (size_t)npen * 4); }
    if (nbias) { memcpy(tk_host + o_bt, bias_tok, (size_t)nbias * 4); memcpy(tk_host + o_bv, bias_val, (size_t)nbias * 4); }
    if (allow_bits) memcpy(tk_host + o_al, allow_bits, (size_t)nrows * words * 4);
    CK(cudaStreamWaitEvent(sm_stream, step_done, 0));
    CK(cudaMemcpyAsync(tk_dev, tk_host, total, cudaMemcpyHostToDevice, sm_stream));
    SampleAdjust a;
    a.slot = (const int*)(tk_dev + o_slot);
    a.pen_off = (const int*)(tk_dev + o_po); a.pen_tok = (const unsigned*)(tk_dev + o_pt); a.pen_val = (const float*)(tk_dev + o_pv);
    a.bias_off = (const int*)(tk_dev + o_bo); a.bias_tok = (const unsigned*)(tk_dev + o_bt); a.bias_val = (const float*)(tk_dev + o_bv);
    a.allow = allow_bits ? (const unsigned*)(tk_dev + o_al) : nullptr;
    return a;
}

void b200rwkv_engine::sample_topk(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok, const float* pen_val,
                                  const uint32_t* allow_bits, const int32_t* bias_off, const uint32_t* bias_tok, const float* bias_val,
                                  int top_k, uint32_t* ids_out, float* probs_out) {
    REQUIRE(rank == 0, B200RWKV_ERR_INVALID, "sample_topk: only rank 0 holds the gathered logits");
    REQUIRE(tk_cand_x, B200RWKV_ERR_UNSUPPORTED, "sample_topk: num_vocab > 65536 is not supported");
    REQUIRE(ids_out && probs_out, B200RWKV_ERR_INVALID, "sample_topk: bad argument");
    REQUIRE(top_k >= 1 && top_k <= TOPK_MAX, B200RWKV_ERR_INVALID, "sample_topk: top_k must be in [1, 128]");
    REQUIRE(top_k <= V, B200RWKV_ERR_INVALID, "sample_topk: top_k exceeds num_vocab");
    check_sample_slots(nrows, slots, "sample_topk");
    check_sample_lists(nrows, pen_off, pen_tok, pen_val, bias_off, bias_tok, bias_val, "sample_topk");
    CK(cudaSetDevice(dev));
    TopkParams tp;
    memset(&tp, 0, sizeof(tp));
    tp.keep = d_keep; tp.V = V; tp.nseg = cdiv(V, TOPK_SEG);
    tp.adj = stage_sample_args(nrows, slots, pen_off, pen_tok, pen_val, allow_bits, bias_off, bias_tok, bias_val);
    tp.cand_x = tk_cand_x; tp.cand_id = tk_cand_id; tp.stats = tk_stats;
    tp.top_k = top_k; tp.out_id = tk_out_id; tp.out_p = tk_out_p;
    topk_segment_kernel<<<dim3(tp.nseg, nrows), TOPK_SEG_THREADS, 0, sm_stream>>>(tp);
    CK(cudaGetLastError());
    topk_merge_kernel<<<nrows, TOPK_MERGE_THREADS, 0, sm_stream>>>(tp);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ids_out, tk_out_id, (size_t)nrows * top_k * 4, cudaMemcpyDeviceToHost, sm_stream));
    CK(cudaMemcpyAsync(probs_out, tk_out_p, (size_t)nrows * top_k * 4, cudaMemcpyDeviceToHost, sm_stream));
    CK(cudaStreamSynchronize(sm_stream));
}

// The whole adjusted distribution of each listed slot's kept row (sample.cuh, probs_*_kernel).  Same thread contract as
// sample_topk; the caller has checked the adjustment lists, probs_out and nrows >= 1.  The kept rows are only read.
void b200rwkv_engine::sample_probs(int nrows, const int32_t* slots, const int32_t* pen_off, const uint32_t* pen_tok, const float* pen_val,
                                   const uint32_t* allow_bits, const int32_t* bias_off, const uint32_t* bias_tok, const float* bias_val,
                                   float* probs_out) {
    REQUIRE(rank == 0, B200RWKV_ERR_INVALID, "sample_probs: only rank 0 holds the gathered logits");
    check_sample_slots(nrows, slots, "sample_probs");
    CK(cudaSetDevice(dev));
    ProbsParams pp;
    memset(&pp, 0, sizeof(pp));
    pp.keep = d_keep; pp.V = V; pp.nseg = cdiv(V, TOPK_SEG); pp.ld = (V + 3) & ~3;
    const size_t row_bytes = (size_t)nrows * pp.ld * 4, need = row_bytes + (size_t)nrows * pp.nseg * sizeof(float2);
    sp_dev.grow(need, std::min(std::max<size_t>(need * 2, 1 << 20), (size_t)S * (pp.ld * 4 + pp.nseg * sizeof(float2))));
    pp.adj = stage_sample_args(nrows, slots, pen_off, pen_tok, pen_val, allow_bits, bias_off, bias_tok, bias_val);
    pp.out = (float*)sp_dev.p;
    pp.stats = (float2*)(sp_dev + row_bytes);
    probs_stats_kernel<<<dim3(pp.nseg, nrows), TOPK_SEG_THREADS, 0, sm_stream>>>(pp);
    CK(cudaGetLastError());
    probs_write_kernel<<<dim3(pp.nseg, nrows), TOPK_SEG_THREADS, 0, sm_stream>>>(pp);
    CK(cudaGetLastError());
    if (pp.ld == V) CK(cudaMemcpyAsync(probs_out, pp.out, row_bytes, cudaMemcpyDeviceToHost, sm_stream));
    else CK(cudaMemcpy2DAsync(probs_out, (size_t)V * 4, pp.out, (size_t)pp.ld * 4, (size_t)V * 4, nrows, cudaMemcpyDeviceToHost, sm_stream));
    CK(cudaStreamSynchronize(sm_stream));
}

// API layout <-> device layout for a live slot (snap == nullptr) or a snapshot record [L][C | Hl*N*N | C]
void b200rwkv_engine::state_xform(int slot, bool import, float* snap) {
    StateXform x;
    const size_t W = (size_t)Hl * N * N;
    x.api = d_api;
    if (snap) {
        const size_t rec = 2 * (size_t)C + W;
        x.att = snap; x.wkv = snap + C; x.ffn = snap + C + W;
        x.att_ls = x.wkv_ls = x.ffn_ls = rec;
    } else {
        x.att = att_shift + (size_t)slot * C; x.att_ls = (size_t)S * C;
        x.ffn = ffn_shift + (size_t)slot * C; x.ffn_ls = (size_t)S * C;
        x.wkv = wkv_state + (size_t)slot * W; x.wkv_ls = (size_t)S * W;
    }
    x.L = L; x.C = C; x.Hl = Hl; x.h0 = rank * Hl; x.transpose = (info.version != 7);
    const size_t total = (size_t)L * (N + 2) * C;
    const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms * 32);
    if (import) state_xform_kernel<true><<<grid, 256, 0, stream>>>(x);
    else state_xform_kernel<false><<<grid, 256, 0, stream>>>(x);
    CK(cudaGetLastError());
}

// =========================================================================================
// in-process tensor-parallel group
// =========================================================================================
void Group::start(int world) {
    status.assign(world, 0);
    errs.assign(world, "");
    for (int r = 1; r < world; ++r)
        workers.emplace_back([this, r]() {
            uint64_t seen = 0;
            for (;;) {
                std::function<int32_t(int)> fn;
                {
                    std::unique_lock<std::mutex> lk(m);
                    cv.wait(lk, [&] { return stop || gen != seen; });
                    if (stop) return;
                    seen = gen;
                    fn = job;
                }
                int32_t st;
                try {
                    st = fn(r);
                } catch (const std::exception& ex) {
                    g_err = ex.what();
                    st = B200RWKV_ERR_INVALID;
                }
                {
                    std::lock_guard<std::mutex> lk(m);
                    status[r] = st;
                    errs[r] = st < 0 ? g_err : std::string();
                    --pending;
                }
                cv.notify_all();
            }
        });
}

void Group::shutdown() {
    {
        std::lock_guard<std::mutex> lk(m);
        stop = true;
    }
    cv.notify_all();
    for (auto& t : workers) t.join();
    workers.clear();
}

// run fn(rank) on every rank at once; the first failure (lowest rank) is what the caller sees
int32_t Group::spmd(const std::function<int32_t(int)>& fn) {
    std::lock_guard<std::mutex> call(call_mu);
    {
        std::lock_guard<std::mutex> lk(m);
        job = fn;
        pending = (int)workers.size();
        ++gen;
    }
    cv.notify_all();
    int32_t st0;
    try {
        st0 = fn(0);
    } catch (const std::exception& ex) {
        g_err = ex.what();
        st0 = B200RWKV_ERR_INVALID;
    }
    {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return pending == 0; });
    }
    if (st0 < 0) return st0;
    for (size_t r = 1; r < status.size(); ++r)
        if (status[r] < 0) {
            g_err = "rank " + std::to_string(r) + ": " + errs[r];
            return status[r];
        }
    return st0;
}

// =========================================================================================
// C ABI
// =========================================================================================
// Error text is thread-local: the reference makes engine calls from two tasks (infer / softmax, run.rs:1232-1237) and a
// per-engine string would race between them.  b200rwkv_last_error() returns the message of the calling thread's last failure.
#define API_BEGIN(e)                            \
    std::string* errp_ = &g_err;                \
    (void)(e);                                  \
    try {
#define API_END                                  \
    }                                            \
    catch (const Error& ex) {                    \
        *errp_ = ex.what();                      \
        return ex.code;                          \
    }                                            \
    catch (const std::exception& ex) {           \
        *errp_ = ex.what();                      \
        return B200RWKV_ERR_INVALID;             \
    }                                            \
    catch (...) {                                \
        *errp_ = "unknown exception";            \
        return B200RWKV_ERR_INVALID;             \
    }                                            \
    return B200RWKV_OK;

// entries that answer a count: the count `body` returns, or the negative status of its failure
template <typename F>
static int32_t api_count(F body) {
    int32_t n = 0;
    const int32_t st = [&]() -> int32_t {
        API_BEGIN((b200rwkv_engine*)nullptr)
        n = body();
        API_END
    }();
    return st < 0 ? st : n;
}

extern "C" {

int32_t b200rwkv_info_from_st(const uint8_t* st, size_t len, b200rwkv_info* out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(out, B200RWKV_ERR_INVALID, "null out");
    StFile f(st, len);
    *out = derive_info(f);
    API_END
}

struct LoraArg { const uint8_t* st; size_t len; float alpha; };

static int32_t create_rank(const uint8_t* st, size_t len, int32_t device, int32_t max_batch, int32_t token_chunk_size,
                           int32_t precision, int32_t rank, int32_t world, const std::vector<LoraArg>& lora, b200rwkv_engine** out,
                           int32_t quant_layers = 0, int32_t quant_type = 0,
                           const std::vector<b200rwkv_engine::LoraSrc>& adapters = {}, int32_t places = 0,
                           uint32_t targets = 0, bool batch_inv = false, bool quant_adapters = false) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(out, B200RWKV_ERR_INVALID, "null out");
    *out = nullptr;
    REQUIRE(precision == 0 || precision == 1, B200RWKV_ERR_INVALID, "precision must be 0 (fp16) or 1 (fp32)");
    REQUIRE(max_batch >= 1 && max_batch <= 1024, B200RWKV_ERR_INVALID, "max_batch out of range");
    REQUIRE(token_chunk_size >= 1, B200RWKV_ERR_INVALID, "token_chunk_size must be >= 1");
    REQUIRE(world >= 1 && world <= 8 && rank >= 0 && rank < world, B200RWKV_ERR_INVALID, "bad rank/world");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    REQUIRE(ce == cudaSuccess && ndev > 0, B200RWKV_ERR_CUDA,
            std::string("no CUDA device (there is no CPU fallback): ") + cudaGetErrorString(ce));
    REQUIRE(device >= 0 && device < ndev, B200RWKV_ERR_INVALID, "device ordinal out of range");
    CK(cudaSetDevice(device));
    watchdog_setup();
    if (g_wd_host) {
        unsigned* dptr = nullptr;
        CK(cudaHostGetDevicePointer(&dptr, g_wd_host, 0));
        CK(cudaMemcpyToSymbol(g_watchdog, &dptr, sizeof(dptr)));
    }
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    REQUIRE(prop.major == 9 && prop.minor == 0, B200RWKV_ERR_UNSUPPORTED,
            "this library is built for sm_90a (H100) only; found sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
    StFile f(st, len);
    std::vector<std::unique_ptr<StFile>> lora_files;
    std::unique_ptr<b200rwkv_engine> e(new b200rwkv_engine());
    for (const LoraArg& la : lora) {
        REQUIRE(la.st && la.len > 8, B200RWKV_ERR_INVALID, "null LoRA image");
        lora_files.emplace_back(new StFile(la.st, la.len));
        e->loras.push_back({lora_files.back().get(), la.alpha});
    }
    e->dev = device; e->rank = rank; e->world = world; e->num_sms = prop.multiProcessorCount;
    e->S = max_batch; e->chunk = token_chunk_size; e->precision = precision;
    REQUIRE(quant_layers >= 0 && quant_type >= 0, B200RWKV_ERR_INVALID, "bad quant_layers / quant_type");
    e->quant_layers = quant_type == QT_NONE ? 0 : quant_layers;
    e->quant_type = quant_layers == 0 ? (int)QT_NONE : quant_type;
    e->adapters = adapters;
    e->n_adapters = adapters.empty() ? places : (int)adapters.size();
    e->ad_targets = targets;
    e->batch_inv = batch_inv;
    e->quant_adapters = quant_adapters;
    e->build(f);
    e->loras.clear();            // the LoRA and adapter images are only borrowed during the build
    e->adapters.clear();
    *out = e.release();
    API_END
}

int32_t b200rwkv_create_tp(const uint8_t* st, size_t len, int32_t device, int32_t max_batch, int32_t token_chunk_size,
                           int32_t precision, int32_t rank, int32_t world, b200rwkv_engine** out) {
    return create_rank(st, len, device, max_batch, token_chunk_size, precision, rank, world, {}, out);
}

int32_t b200rwkv_create(const uint8_t* st, size_t len, int32_t device, int32_t max_batch, int32_t token_chunk_size,
                        int32_t precision, b200rwkv_engine** out) {
    return create_rank(st, len, device, max_batch, token_chunk_size, precision, 0, 1, {}, out);
}

struct TpHandle {            // wire format of the 128-byte blob
    cudaIpcMemHandle_t ipc;  // 64 bytes
    int32_t rank, world;
    uint64_t comm_bytes;
    int32_t pid;
    int32_t device;
};
static_assert(sizeof(TpHandle) <= B200RWKV_TP_HANDLE_BYTES, "handle blob too large");

int32_t b200rwkv_tp_export(b200rwkv_engine* e, uint8_t* handle_out) {
    API_BEGIN(e)
    REQUIRE(e && handle_out, B200RWKV_ERR_INVALID, "null argument");
    CK(cudaSetDevice(e->dev));
    TpHandle h;
    memset(&h, 0, sizeof(h));
    CK(cudaIpcGetMemHandle(&h.ipc, e->comm_base));
    h.rank = e->rank; h.world = e->world; h.comm_bytes = e->comm_bytes; h.pid = (int32_t)getpid(); h.device = e->dev;
    memset(handle_out, 0, B200RWKV_TP_HANDLE_BYTES);
    memcpy(handle_out, &h, sizeof(h));
    API_END
}

int32_t b200rwkv_tp_connect(b200rwkv_engine* e, const uint8_t* handles) {
    API_BEGIN(e)
    REQUIRE(e && handles, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(!e->connected || e->world == 1, B200RWKV_ERR_INVALID, "already connected");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    for (int q = 0; q < e->world; ++q) {
        TpHandle h;
        memcpy(&h, handles + (size_t)q * B200RWKV_TP_HANDLE_BYTES, sizeof(h));
        REQUIRE(h.rank == q && h.world == e->world && h.comm_bytes == e->comm_bytes, B200RWKV_ERR_INVALID,
                "tp_connect: handle blobs are not rank-ordered or come from a different model/world");
        if (q == e->rank) {
            e->peer_base[q] = e->comm_base;
        } else {
            void* p = nullptr;
            CK(cudaIpcOpenMemHandle(&p, h.ipc, cudaIpcMemLazyEnablePeerAccess));
            e->peer_base[q] = (uint8_t*)p;
            e->peer_ipc[q] = true;
        }
    }
    e->finalize_tp();
    CK(cudaDeviceSynchronize());
    API_END
}

// In-process variant (all ranks live in this process, e.g. tests with several ranks on one GPU, or a
// host that owns every GPU of the box as in SURVEY.md §8b): exchange the comm-block pointers directly.
int32_t b200rwkv_tp_connect_local(b200rwkv_engine** engines, int32_t n) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(engines && n >= 1 && n <= 8, B200RWKV_ERR_INVALID, "bad argument");
    for (int i = 0; i < n; ++i)
        REQUIRE(engines[i] && engines[i]->world == n && engines[i]->rank == i && engines[i]->comm_bytes == engines[0]->comm_bytes,
                B200RWKV_ERR_INVALID, "tp_connect_local: engines must be rank-ordered ranks of one world");
    for (int i = 0; i < n; ++i) {
        b200rwkv_engine* e = engines[i];
        CK(cudaSetDevice(e->dev));
        for (int q = 0; q < n; ++q) {
            if (engines[q]->dev != e->dev) {
                int can = 0;
                CK(cudaDeviceCanAccessPeer(&can, e->dev, engines[q]->dev));
                REQUIRE(can, B200RWKV_ERR_CUDA, "no peer access between the devices");
                cudaError_t pe = cudaDeviceEnablePeerAccess(engines[q]->dev, 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CK(pe);
                (void)cudaGetLastError();
            }
            e->peer_base[q] = engines[q]->comm_base;
        }
        e->finalize_tp();
        CK(cudaDeviceSynchronize());
    }
    API_END
}

void b200rwkv_destroy(b200rwkv_engine* e) {
    if (!e) return;
    if (e->group) {
        std::unique_ptr<Group> g = std::move(e->group);
        g->shutdown();
        for (size_t r = 1; r < g->ranks.size(); ++r) delete g->ranks[r];
    }
    delete e;
}

int32_t b200rwkv_get_info(b200rwkv_engine* e, b200rwkv_info* out) {
    API_BEGIN(e)
    REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
    *out = e->info;
    API_END
}

static int32_t rank_infer(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const int32_t* ntok, const uint32_t* tokens,
                       const int32_t* option, float* logits_out, size_t logits_cap, int32_t* rows_out,
                       const b200rwkv_engine::ScoreOut* score = nullptr, const b200rwkv_engine::SnapPlan* snap = nullptr) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    e->infer(nslot, slot, ntok, tokens, option, logits_out, logits_cap, rows_out, score, snap);
    API_END
}

int32_t b200rwkv_state_shape(b200rwkv_engine* e, int64_t shape[4]) {
    API_BEGIN(e)
    REQUIRE(e && shape, B200RWKV_ERR_INVALID, "null argument");
    shape[0] = e->C; shape[1] = e->N + 2; shape[2] = e->L; shape[3] = 1;
    API_END
}

int32_t b200rwkv_state_init(b200rwkv_engine* e, float* out) {
    API_BEGIN(e)
    REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    if (e->init_state.empty()) memset(out, 0, n * 4);
    else memcpy(out, e->init_state.data(), n * 4);
    API_END
}

static int32_t rank_state_load(b200rwkv_engine* e, int32_t slot, const float* in) {
    API_BEGIN(e)
    REQUIRE(e && in, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(slot >= 0 && slot < e->S, B200RWKV_ERR_STATE, "slot out of range");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    CK(cudaMemcpyAsync(e->d_api, in, n * 4, cudaMemcpyHostToDevice, e->stream));
    e->state_xform(slot, true);
    CK(cudaStreamSynchronize(e->stream));
    {       // a host state carries no logits row: the slot's kept row belonged to the state just replaced
        std::lock_guard<std::mutex> lk2(e->keep_mu);
        e->keep_valid[slot] = 0;
    }
    API_END
}

static int32_t rank_state_back(b200rwkv_engine* e, int32_t slot, float* out) {
    API_BEGIN(e)
    REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(slot >= 0 && slot < e->S, B200RWKV_ERR_STATE, "slot out of range");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    e->state_xform(slot, false);
    CK(cudaMemcpyAsync(out, e->d_api, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    API_END
}

// device-side snapshot: [L][C | Hl*N*N | C]
static void snapshot_copy(b200rwkv_engine* e, int slot, float* buf, bool to_snapshot) {
    const size_t C = e->C, W = (size_t)e->Hl * e->N * e->N, S = e->S, L = e->L;
    const size_t rec = 2 * C + W;
    struct Part { float* dev; size_t width; size_t off; };
    Part parts[3] = {{e->att_shift + (size_t)slot * C, C, 0}, {e->wkv_state + (size_t)slot * W, W, C}, {e->ffn_shift + (size_t)slot * C, C, C + W}};
    for (auto& p : parts) {
        if (to_snapshot)
            CK(cudaMemcpy2DAsync(buf + p.off, rec * 4, p.dev, S * p.width * 4, p.width * 4, L, cudaMemcpyDeviceToDevice, e->stream));
        else
            CK(cudaMemcpy2DAsync(p.dev, S * p.width * 4, buf + p.off, rec * 4, p.width * 4, L, cudaMemcpyDeviceToDevice, e->stream));
    }
}


static int32_t rank_state_read(b200rwkv_engine* e, int32_t slot, uint64_t* snapshot_id) {
    API_BEGIN(e)
    REQUIRE(e && snapshot_id, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(slot >= 0 && slot < e->S, B200RWKV_ERR_STATE, "slot out of range");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    bool has_row;
    {
        std::lock_guard<std::mutex> lk2(e->keep_mu);
        has_row = e->d_keep && e->keep_valid[slot];
    }
    Snapshot sn = snapshot_alloc(e, has_row);
    snapshot_copy(e, slot, sn.buf, true);
    // the slot's last logits row travels with the state (CachedItem.output, run.rs:199-205): a cache hit can be sampled
    // on the device without re-running the last token
    if (has_row) CK(cudaMemcpyAsync(sn.logits, e->d_keep + (size_t)slot * e->V, (size_t)e->V * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    const uint64_t id = e->next_snap++;
    e->snaps[id] = std::move(sn);
    *snapshot_id = id;
    API_END
}

static int32_t rank_state_write(b200rwkv_engine* e, int32_t slot, uint64_t snapshot_id) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(slot >= 0 && slot < e->S, B200RWKV_ERR_STATE, "slot out of range");
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->snaps.find(snapshot_id);
    REQUIRE(it != e->snaps.end(), B200RWKV_ERR_STATE, "unknown snapshot id");
    CK(cudaSetDevice(e->dev));
    snapshot_copy(e, slot, it->second.buf, false);
    if (e->d_keep && it->second.logits)
        CK(cudaMemcpyAsync(e->d_keep + (size_t)slot * e->V, it->second.logits, (size_t)e->V * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaEventRecord(e->step_done, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    {
        std::lock_guard<std::mutex> lk2(e->keep_mu);
        e->keep_valid[slot] = (e->d_keep && it->second.logits) ? 1 : 0;
    }
    API_END
}

static int32_t rank_state_free(b200rwkv_engine* e, uint64_t snapshot_id) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->snaps.find(snapshot_id);
    REQUIRE(it != e->snaps.end(), B200RWKV_ERR_STATE, "unknown snapshot id");
    CK(cudaSetDevice(e->dev));
    e->snaps.erase(it);
    API_END
}

// ---- device-resident state cache (SURVEY.md §8f-4): snapshots <-> host tensors, without passing through a slot ----
static int32_t rank_snapshot_back(b200rwkv_engine* e, uint64_t snapshot_id, float* state_out, float* logits_out) {
    API_BEGIN(e)
    REQUIRE(e && (state_out || logits_out), B200RWKV_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->snaps.find(snapshot_id);
    REQUIRE(it != e->snaps.end(), B200RWKV_ERR_STATE, "unknown snapshot id");
    CK(cudaSetDevice(e->dev));
    if (state_out) {
        const size_t n = (size_t)e->L * (e->N + 2) * e->C;
        e->state_xform(0, false, it->second.buf);
        CK(cudaMemcpyAsync(state_out, e->d_api, n * 4, cudaMemcpyDeviceToHost, e->stream));
    }
    if (logits_out) {
        REQUIRE(it->second.logits, B200RWKV_ERR_STATE, "snapshot holds no logits row");
        CK(cudaMemcpyAsync(logits_out, it->second.logits, (size_t)e->V * 4, cudaMemcpyDeviceToHost, e->stream));
    }
    CK(cudaStreamSynchronize(e->stream));
    API_END
}

static int32_t rank_snapshot_load(b200rwkv_engine* e, const float* state_in, const float* logits_in, uint64_t* snapshot_id) {
    API_BEGIN(e)
    REQUIRE(e && state_in && snapshot_id, B200RWKV_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    Snapshot sn = snapshot_alloc(e, logits_in != nullptr && e->d_keep != nullptr);
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    CK(cudaMemcpyAsync(e->d_api, state_in, n * 4, cudaMemcpyHostToDevice, e->stream));
    e->state_xform(0, true, sn.buf);
    if (sn.logits) CK(cudaMemcpyAsync(sn.logits, logits_in, (size_t)e->V * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    const uint64_t id = e->next_snap++;
    e->snaps[id] = std::move(sn);
    *snapshot_id = id;
    API_END
}

int32_t b200rwkv_cache_stats(b200rwkv_engine* e, int64_t* num_snapshots, int64_t* bytes_used, int64_t* bytes_free) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    int64_t used = 0;
    for (auto& kv : e->snaps) used += (int64_t)(kv.second.buf.bytes + kv.second.logits.bytes);
    size_t fr = 0, tot = 0;
    CK(cudaMemGetInfo(&fr, &tot));
    if (num_snapshots) *num_snapshots = (int64_t)e->snaps.size();
    if (bytes_used) *bytes_used = used;
    if (bytes_free) *bytes_free = (int64_t)fr;
    API_END
}

// `vN::read_state(&context, &info, reader)` (reference lib.rs:378-389; `.state` files and InputState::File, run.rs:403-437):
// host only.  out: [L][N+2][C] f32 in the web-rwkv state layout.
int32_t b200rwkv_read_state(const b200rwkv_info* info, const uint8_t* st, size_t len, float* out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(info && out, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(info->num_layer > 0 && info->num_head > 0 && info->head_size > 0 && info->num_emb == info->num_head * info->head_size,
            B200RWKV_ERR_INVALID, "bad model info");
    StFile f(st, len);
    std::vector<float> v;
    REQUIRE(state_from_st(f, info->num_layer, info->num_head, info->head_size, info->num_emb, v), B200RWKV_ERR_INVALID,
            "no blocks.*.att.time_state tensors in this file");
    memcpy(out, v.data(), v.size() * 4);
    API_END
}

int32_t b200rwkv_softmax(b200rwkv_engine* e, int32_t rows, const float* in, float* out) {
    API_BEGIN(e)
    REQUIRE(e && (rows == 0 || (in && out)) && rows >= 0, B200RWKV_ERR_INVALID, "bad argument");
    if (rows == 0) return B200RWKV_OK;
    std::lock_guard<std::mutex> lk(e->sm_mu);
    CK(cudaSetDevice(e->dev));
    const size_t bytes = (size_t)rows * e->V * 4;
    e->sm_in.grow(bytes, bytes);
    e->sm_out.grow(bytes, bytes);
    CK(cudaMemcpyAsync(e->sm_in, in, bytes, cudaMemcpyHostToDevice, e->sm_stream));
    softmax_kernel<<<rows, 1024, 0, e->sm_stream>>>(e->sm_in, e->sm_out, e->V);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, e->sm_out, bytes, cudaMemcpyDeviceToHost, e->sm_stream));
    CK(cudaStreamSynchronize(e->sm_stream));
    API_END
}

int32_t b200rwkv_sample_topk(b200rwkv_engine* e, int32_t nrows, const int32_t* slots, const int32_t* penalty_offset,
                             const uint32_t* penalty_token, const float* penalty_value, const uint32_t* allow_bits,
                             const int32_t* bias_offset, const uint32_t* bias_token, const float* bias_value, int32_t top_k,
                             uint32_t* ids_out, float* probs_out) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->sm_mu);
    e->sample_topk(nrows, slots, penalty_offset, penalty_token, penalty_value, allow_bits, bias_offset, bias_token, bias_value, top_k,
                   ids_out, probs_out);
    API_END
}

int32_t b200rwkv_sample_probs(b200rwkv_engine* e, int32_t nrows, const int32_t* slots, const int32_t* penalty_offset,
                              const uint32_t* penalty_token, const float* penalty_value, const uint32_t* allow_bits,
                              const int32_t* bias_offset, const uint32_t* bias_token, const float* bias_value, float* probs_out) {
    API_BEGIN(e)
    REQUIRE(nrows >= 1 && slots && probs_out, B200RWKV_ERR_INVALID, "sample_probs: bad argument");
    REQUIRE(!e || nrows <= e->S, B200RWKV_ERR_INVALID, "sample_probs: nrows exceeds max_batch");
    check_sample_lists(nrows, penalty_offset, penalty_token, penalty_value, bias_offset, bias_token, bias_value, "sample_probs");
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->sm_mu);
    e->sample_probs(nrows, slots, penalty_offset, penalty_token, penalty_value, allow_bits, bias_offset, bias_token, bias_value, probs_out);
    API_END
}

int32_t b200rwkv_host_alloc(size_t bytes, void** out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(out, B200RWKV_ERR_INVALID, "null out");
    CK(cudaMallocHost(out, bytes));
    API_END
}

void b200rwkv_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

// The arguments of the decode routes (bench_decode, profile_step, profile_insitu), before any CUDA call, as infer checks its
// entries: nslot in [1, min(S, maxT)], slots in [0, S) (ERR_STATE) and distinct (two WKV CTAs would read-modify-write one
// state), token ids below V for all `nsteps` steps.
static void check_decode_args(const b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int nsteps,
                              const char* what) {
    const std::string w(what);
    REQUIRE(nslot >= 1 && nslot <= e->S && nslot <= e->maxT, B200RWKV_ERR_INVALID, w + ": nslot outside [1, max_batch]");
    std::vector<char> seen(e->S, 0);
    for (int i = 0; i < nslot; ++i) {
        REQUIRE(slot[i] >= 0 && slot[i] < e->S, B200RWKV_ERR_STATE, w + ": slot " + std::to_string(slot[i]) + " out of range");
        REQUIRE(!seen[slot[i]], B200RWKV_ERR_INVALID, w + ": duplicate slot " + std::to_string(slot[i]));
        seen[slot[i]] = 1;
    }
    for (size_t i = 0; i < (size_t)nsteps * nslot; ++i)
        REQUIRE(tokens[i] < (uint32_t)e->V, B200RWKV_ERR_INVALID, w + ": token id outside the vocabulary");
}

// A profiling step moves the listed slots' states on without writing their kept rows (it runs no enqueue_keep): drop them,
// as infer does for a NONE entry with tokens.
static void drop_kept_rows(b200rwkv_engine* e, int32_t nslot, const int32_t* slot) {
    std::lock_guard<std::mutex> lk(e->keep_mu);
    for (int i = 0; i < nslot; ++i) e->keep_valid[slot[i]] = 0;
}

static void build_decode_metas(b200rwkv_engine* e, int nslot, const int32_t* slot, const uint32_t* tokens, int nsteps,
                               std::vector<int>& all) {
    all.assign((size_t)nsteps * e->meta_ints, 0);
    std::vector<int> s_slots(slot, slot + nslot), s_counts(nslot, 1), s_out(nslot, 1);
    std::vector<const uint32_t*> s_toks(nslot);
    for (int st = 0; st < nsteps; ++st) {
        for (int i = 0; i < nslot; ++i) s_toks[i] = tokens + (size_t)st * nslot + i;
        int R = 0;
        e->fill_meta(all.data() + (size_t)st * e->meta_ints, s_slots, s_counts, s_toks, s_out, &R);
    }
}

static int32_t rank_bench_decode(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int32_t warmup,
                              int32_t steps, int32_t flush_l2, float* ms_out, int64_t* launches_out, float* step_ms_out) {
    API_BEGIN(e)
    REQUIRE(e && slot && tokens && ms_out, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(steps >= 1 && warmup >= 0, B200RWKV_ERR_INVALID, "bench_decode: bad step count");
    const int nsteps = warmup + steps;
    check_decode_args(e, nslot, slot, tokens, nsteps, "bench_decode");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    std::vector<int> all;
    build_decode_metas(e, nslot, slot, tokens, nsteps, all);
    long long launches_before = 0;
    Buf<int> d_all(all.size() * 4);
    CK(cudaMemcpy(d_all, all.data(), all.size() * 4, cudaMemcpyHostToDevice));
    Buf<void> flush;
    const size_t flush_bytes = 256u << 20;
    if (flush_l2) flush = Buf<void>(flush_bytes);
    Event ea = new_event(), eb = new_event();
    std::vector<Event> marks;                  // per-step boundaries (optional): the distribution of the step time
    if (step_ms_out)
        for (int i = 0; i < steps; ++i) marks.push_back(new_event());
    StepShape sh = e->step_shape(nslot, nslot);
    sh.ad = e->step_bound(std::vector<int>(slot, slot + nslot));
    for (int st = 0; st < nsteps; ++st) {
        if (st == warmup) {
            CK(cudaStreamSynchronize(e->stream));
            CK(cudaEventRecord(ea, e->stream));
            launches_before = e->launch_total;
        }
        if (flush) CK(cudaMemsetAsync(flush, st & 0xff, flush_bytes, e->stream));
        CK(cudaMemcpyAsync(e->d_meta, d_all + (size_t)st * e->meta_ints, e->meta_ints * 4, cudaMemcpyDeviceToDevice, e->stream));
        e->run_step(sh);
        if (step_ms_out && st >= warmup) CK(cudaEventRecord(marks[st - warmup], e->stream));
    }
    CK(cudaEventRecord(eb, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (e->d_keep && e->rank == 0) {          // every step kept each slot's logits row (enqueue_keep): sample_topk may read it
        std::lock_guard<std::mutex> lk2(e->keep_mu);
        for (int i = 0; i < nslot; ++i) e->keep_valid[slot[i]] = 1;
    }
    CK(cudaEventElapsedTime(ms_out, ea, eb));
    for (int i = 0; i < (int)marks.size(); ++i) {
        CK(cudaEventElapsedTime(step_ms_out + i, i == 0 ? ea : marks[i - 1], marks[i]));
    }
    if (launches_out) *launches_out = (int64_t)(e->launch_total - launches_before);
    API_END
}

static int32_t rank_profile_step(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, float ms[4],
                              int32_t launches[4], int64_t* gemm_weight_bytes) {
    API_BEGIN(e)
    REQUIRE(e && slot && tokens && ms && launches, B200RWKV_ERR_INVALID, "null argument");
    check_decode_args(e, nslot, slot, tokens, 1, "profile_step");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    std::vector<int> all;
    build_decode_metas(e, nslot, slot, tokens, 1, all);
    CK(cudaMemcpyAsync(e->d_meta, all.data(), e->meta_ints * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    drop_kept_rows(e, nslot, slot);
    Profiler prof;
    StepShape sh = e->step_shape(nslot, nslot);
    sh.ad = e->step_bound(std::vector<int>(slot, slot + nslot));      // bound slots: the adapter plans and their shrinks
    e->enqueue_step(e->stream, sh, &prof);
    CK(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < 4; ++i) { ms[i] = 0.f; launches[i] = 0; }
    for (auto& r : prof.recs) {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, r.a, r.b));
        ms[r.cls] += t;
        launches[r.cls] += 1;
    }
    if (gemm_weight_bytes) *gemm_weight_bytes = (int64_t)prof.weight_bytes;
    API_END
}

// In-situ timeline of a graph-replayed decode step: every launch of the step writes globaltimer stamps (CTA 0: entry, past
// griddepcontrol.wait, exit; projections: exit of EVERY CTA).  A launch's window is [released by griddepcontrol.wait, last CTA
// exit]: with programmatic dependent launch a kernel is resident long before it may touch its inputs, so CUDA events around
// launches (b200rwkv_profile_step) over-count; windows of consecutive launches cannot overlap (the wait returns only when the
// previous grid has completed), so their sum is <= the step.  Averages over `reps` replays of a traced copy of the step graph.
static int32_t rank_profile_insitu(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int32_t reps,
                                int32_t cap, int32_t* n_out, int32_t* types, double* start_us, double* end_us, int64_t* bytes,
                                double* step_us) {
    API_BEGIN(e)
    REQUIRE(e && slot && tokens && n_out && types && start_us && end_us && bytes && step_us && reps >= 1 && cap >= 1, B200RWKV_ERR_INVALID,
            "bad argument");
    check_decode_args(e, nslot, slot, tokens, 1, "profile_insitu");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    if (!e->d_step_trace) e->d_step_trace = (unsigned long long*)e->dalloc((size_t)b200rwkv_engine::STEP_TRACE_MAX * b200rwkv_engine::STEP_TRACE_ROW * 8, true);
    std::vector<int> all;
    build_decode_metas(e, nslot, slot, tokens, 1, all);
    CK(cudaMemcpyAsync(e->d_meta, all.data(), e->meta_ints * 4, cudaMemcpyHostToDevice, e->stream));
    drop_kept_rows(e, nslot, slot);
    StepShape sh = e->step_shape(nslot, nslot);
    sh.ad = e->step_bound(std::vector<int>(slot, slot + nslot));
    // traced copy of the step graph (the production graphs carry null trace pointers)
    e->step_trace_types.clear();
    e->step_trace_bytes.clear();
    const GraphExec ge = capture_graph(e->stream, [&] {
        e->trace_capture = true;
        struct Off { bool& f; ~Off() { f = false; } } off{e->trace_capture};     // on every exit
        e->enqueue_step(e->stream, sh, nullptr);
    });
    const int n = (int)e->step_trace_types.size();
    const size_t row = b200rwkv_engine::STEP_TRACE_ROW;
    std::vector<unsigned long long> h((size_t)n * row);
    std::vector<double> s_acc(n, 0.0), e_acc(n, 0.0);
    double step_acc = 0.0;
    e->step_trace_bytes.resize(n, 0);
    for (int r = 0; r < reps + 1; ++r) {        // first replay is warm-up
        CK(cudaMemsetAsync(e->d_step_trace, 0, (size_t)n * row * 8, e->stream));
        CK(cudaGraphLaunch(ge, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        if (r == 0) continue;
        CK(cudaMemcpy(h.data(), e->d_step_trace, (size_t)n * row * 8, cudaMemcpyDeviceToHost));
        unsigned long long t0 = ~0ull, t1 = 0;
        for (int i = 0; i < n; ++i) {
            const unsigned long long* q = h.data() + (size_t)i * row;
            if (q[0] && q[0] < t0) t0 = q[0];
        }
        for (int i = 0; i < n; ++i) {
            const unsigned long long* q = h.data() + (size_t)i * row;
            const bool gemm = e->step_trace_types[i] >= 1000000;
            unsigned long long st = gemm ? q[2] : q[1], en = q[7];
            if (gemm)
                for (int c = 0; c < e->num_sms && 8 + 3 * c + 2 < (int)row; ++c) en = std::max(en, q[8 + 3 * c + 2]);
            if (!st || !en) continue;
            s_acc[i] += (double)(st - t0) * 1e-3;
            e_acc[i] += (double)(en - t0) * 1e-3;
            t1 = std::max(t1, en);
        }
        step_acc += (double)(t1 - t0) * 1e-3;
    }
    int m = 0;
    for (int i = 0; i < n && m < cap; ++i) {
        if (e_acc[i] <= 0.0) continue;
        types[m] = e->step_trace_types[i];
        start_us[m] = s_acc[i] / reps;
        end_us[m] = e_acc[i] / reps;
        bytes[m] = e->step_trace_bytes[i];
        ++m;
    }
    *n_out = m;
    *step_us = step_acc / reps;
    API_END
}

// The quantisers' code blocks on the host, untiled: blocks [tiles][KB] (q_block_bytes(qt) each) into one code per byte,
// codes [rows][KB * 128] for rows < `rows` (<= tiles * 128: padding rows included up to there), and the block parameters:
// Int8 / Int4 p0 = min, p1 = scale [rows][KB]; NF4 p0 = absmax [rows][2 KB].  FP8 blocks hold codes only (its row scales
// are apart).  b200rwkv_op_quantize and b200rwkv_debug_fill both read blocks through this, so the layout oracle/quant_numpy.py,
// tests/fp8_oracle.py and tests/int4_oracle.py are compared with is one.
static void untile_codes(int qt, const uint8_t* h, int tiles, int KB, int rows, uint8_t* codes, uint16_t* p0, uint16_t* p1) {
    const size_t blk = (size_t)q_block_bytes(qt), K = (size_t)KB * GEMM_BK;
    for (int n = 0; n < rows; ++n) {
        const int tile = n / GEMM_BN, r = n % GEMM_BN;
        for (int kb = 0; kb < KB; ++kb) {
            const uint8_t* b = h + ((size_t)tile * KB + kb) * blk;
            uint8_t* c = codes + n * K + (size_t)kb * GEMM_BK;
            if (qt == QT_FP8) {
                for (int k = 0; k < GEMM_BK; ++k) c[k] = b[fp8_code_offset(r, k)];
            } else if (qt == QT_INT8) {
                for (int k = 0; k < GEMM_BK; ++k) c[k] = b[(size_t)((k >> 4) * GEMM_BN + r) * 16 + (k & 15)];
                uint16_t pr[2];
                memcpy(pr, b + GEMM_BN * GEMM_BK + r * 4, 4);
                p1[(size_t)n * KB + kb] = pr[0];      // scale
                p0[(size_t)n * KB + kb] = pr[1];      // min
            } else if (qt == QT_INT4) {
                for (int k = 0; k < GEMM_BK; ++k) {
                    const int nib = int4_nibble(r, k);
                    c[k] = (b[nib >> 1] >> (4 * (nib & 1))) & 15;
                }
                uint16_t pr[2];
                memcpy(pr, b + int4_param_offset(r), 4);
                p1[(size_t)n * KB + kb] = pr[0];      // scale
                p0[(size_t)n * KB + kb] = pr[1];      // min
            } else {
                for (int k = 0; k < GEMM_BK; ++k) {
                    const uint8_t by = b[(size_t)((k >> 5) * GEMM_BN + r) * 16 + ((k & 31) >> 1)];
                    c[k] = (k & 1) ? (by >> 4) : (by & 15);
                }
                uint16_t pr[2];
                memcpy(pr, b + GEMM_BN * GEMM_BK / 2 + r * 4, 4);
                p0[(size_t)n * (2 * KB) + 2 * kb] = pr[0];
                p0[(size_t)n * (2 * KB) + 2 * kb + 1] = pr[1];
            }
        }
    }
}

// f16 weight blocks on the host, untiled: blocks kb0 .. kb0 + nkb - 1 of every tile row of [tiles][stride_kb] blocks
// (repack_weight_kernel's layout: row r, column k of a block at half ((k / 8) * 128 + r) * 8 + k % 8) into
// [tiles * 128][nkb * 128] rows
static void untile_f16(const uint16_t* h, int tiles, int stride_kb, int kb0, int nkb, uint16_t* out) {
    const size_t ld = (size_t)nkb * GEMM_BK, bh = GEMM_WBYTES / 2;
    for (int tile = 0; tile < tiles; ++tile)
        for (int kb = 0; kb < nkb; ++kb) {
            const uint16_t* b = h + ((size_t)tile * stride_kb + kb0 + kb) * bh;
            for (int r = 0; r < GEMM_BN; ++r)
                for (int k = 0; k < GEMM_BK; ++k)
                    out[((size_t)tile * GEMM_BN + r) * ld + (size_t)kb * GEMM_BK + k] = b[((k >> 3) * GEMM_BN + r) * 8 + (k & 7)];
        }
}

// Operator-level entry for the parity tests: the load-time quantiser (qgemm.cuh, fp8gemm.cuh, int4gemm.cuh) on one matrix,
// un-tiled on the host (untile_codes) into plain row-major codes and per-block (per-row for FP8) parameters so that
// oracle/quant_numpy.py, tests/fp8_oracle.py and tests/int4_oracle.py can be compared bit for bit.
int32_t b200rwkv_op_quantize(int32_t device, int32_t quant_type, int32_t N, int32_t K, const uint16_t* w_f16, uint8_t* codes,
                             uint16_t* p0, uint16_t* p1) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(quant_type == QT_INT8 || quant_type == QT_NF4 || quant_type == QT_FP8 || quant_type == QT_INT4, B200RWKV_ERR_UNSUPPORTED,
            "quant_type must be Int8, NF4, FP8 or Int4");
    REQUIRE(N >= 1 && K >= GEMM_BK && K % GEMM_BK == 0 && (size_t)N * K <= ((size_t)1 << 31) && w_f16 && codes && p0, B200RWKV_ERR_INVALID, "bad argument");
    REQUIRE((quant_type != QT_INT8 && quant_type != QT_INT4) || p1, B200RWKV_ERR_INVALID, "Int8 / Int4 need p1 (scales)");
    CK(cudaSetDevice(device));
    const int tiles = cdiv(N, GEMM_BN), KB = K / GEMM_BK;
    const size_t blk = (size_t)q_block_bytes(quant_type), total = (size_t)tiles * KB * blk;
    Buf<__half> src((size_t)N * K * 2);
    Buf<uint8_t> dst(total);
    CK(cudaMemcpy(src, w_f16, (size_t)N * K * 2, cudaMemcpyHostToDevice));
    const size_t nwarp = (size_t)tiles * KB * GEMM_BN;
    int nsm = 0;
    CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    const int grid = (int)std::min<size_t>((nwarp + 7) / 8, (size_t)nsm * 32);
    Buf<float> scales;
    if (quant_type == QT_FP8) {
        scales = Buf<float>((size_t)tiles * FP8_SCALE_BYTES);
        quantize_fp8_kernel<<<std::min(cdiv(tiles * GEMM_BN, 8), nsm * 32), 256>>>(src, K, 0, 0, N, tiles, KB, dst, scales);
    } else if (quant_type == QT_INT8) quantize_weight_kernel<QT_INT8><<<grid, 256>>>(src, K, 0, 0, N, tiles, KB, dst);
    else if (quant_type == QT_INT4) quantize_int4_kernel<<<grid, 256>>>(src, K, 0, 0, N, tiles, KB, dst);
    else quantize_weight_kernel<QT_NF4><<<grid, 256>>>(src, K, 0, 0, N, tiles, KB, dst);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<uint8_t> h(total);
    CK(cudaMemcpy(h.data(), dst, total, cudaMemcpyDeviceToHost));
    if (quant_type == QT_FP8) CK(cudaMemcpy(p0, scales, (size_t)N * 4, cudaMemcpyDeviceToHost));
    untile_codes(quant_type, h.data(), tiles, KB, N, codes, p0, p1);
    API_END
}

// The snapshot arguments of b200rwkv_op_wkv / op_ln, before any CUDA call: distinct token rows of a step of T tokens, and
// records of snap_ld cells that hold `need` cells from snap_off on.  The kernels store records in float4 vectors, so every
// record part starts on a 16-byte boundary: snap_off and snap_ld are multiples of 4.
static void snap_args_ok(int nsnap, const int32_t* tok, const float* rec, int64_t ld, int64_t off, int64_t need, int T) {
    REQUIRE(nsnap >= 0, B200RWKV_ERR_INVALID, "nsnap must be >= 0");
    if (nsnap == 0) return;
    REQUIRE(tok && rec, B200RWKV_ERR_INVALID, "snapshots need snap_tok and snap_rec");
    REQUIRE(off >= 0 && ld >= need && off <= ld - need, B200RWKV_ERR_INVALID, "snap_ld must be >= snap_off + the recorded part");
    REQUIRE(off % 4 == 0 && ld % 4 == 0, B200RWKV_ERR_INVALID, "snap_off and snap_ld must be multiples of 4 (float4 stores)");
    std::vector<char> seen(T, 0);
    for (int k = 0; k < nsnap; ++k) {
        REQUIRE(tok[k] >= 0 && tok[k] < T, B200RWKV_ERR_INVALID, "snapshot token outside [0, T)");
        REQUIRE(!seen[tok[k]], B200RWKV_ERR_INVALID, "snapshot token listed twice");
        seen[tok[k]] = 1;
    }
}

// The step under an operator-level entry (b200rwkv_op_wkv / op_ln / op_gemm).  The constructor checks the step's entries
// (slot, token count) before any CUDA call; start() makes a temporary engine object with the step's pool size and precision,
// one metadata block per launch from its fill_meta and the step's shape from its step_shape: what a step of these entries
// derives.
struct OpStep {
    int S, T = 0, R = 0;
    bool split;
    std::vector<int> slots, counts;
    std::unique_ptr<b200rwkv_engine> e;
    std::vector<int*> metas;                       // device, one per launch; e->d_meta is the first
    std::vector<int> meta0;                        // host copy of the first
    StepShape sh{};
    MetaView snap_meta{};                          // snap_start(): the snapshot block's metadata and record table
    float* const* snap_table = nullptr;

    OpStep(int S_, int nslot, const int32_t* slot, const int32_t* count, int precision) : S(S_), split(precision == 1) {
        REQUIRE(S >= 1 && S <= 1024, B200RWKV_ERR_INVALID, "S must be 1..1024 (max_batch)");
        REQUIRE(nslot >= 1 && nslot <= S && slot && count, B200RWKV_ERR_INVALID, "nslot must be 1..S with slot and count");
        REQUIRE(precision == 0 || precision == 1, B200RWKV_ERR_INVALID, "precision must be 0 or 1");
        std::vector<char> seen(S, 0);
        for (int i = 0; i < nslot; ++i) {
            REQUIRE(slot[i] >= 0 && slot[i] < S, B200RWKV_ERR_STATE, "slot out of range");
            REQUIRE(!seen[slot[i]], B200RWKV_ERR_INVALID, "duplicate slot in one step");
            seen[slot[i]] = 1;
            REQUIRE(count[i] >= 1 && count[i] <= A16_MAX_ROWS - T, B200RWKV_ERR_INVALID, "counts must be >= 1 and sum to <= 128");
            T += count[i];
        }
        REQUIRE(!split || T <= 16, B200RWKV_ERR_UNSUPPORTED, "precision 1 runs decode-shaped steps (T <= 16)");
        slots.assign(slot, slot + nslot);
        counts.assign(count, count + nslot);
    }
    // tokens: [launches][T] ids, or null for id 0; outmode: fill_meta's, per entry
    void start(int device, int launches, const uint32_t* tokens, const std::vector<int>& outmode) {
        CK(cudaSetDevice(device));
        e.reset(new b200rwkv_engine());
        e->dev = device;
        e->S = S;                                  // e->maxT stays A16_MAX_ROWS: the metadata layout of every engine
        e->split_on = split;
        e->stream = new_stream();
        for (int l = 0; l < launches; ++l) {
            std::vector<uint32_t> tk(A16_MAX_ROWS, 0);
            if (tokens) std::copy(tokens + (size_t)l * T, tokens + (size_t)(l + 1) * T, tk.begin());
            std::vector<const uint32_t*> toks(slots.size());
            for (size_t i = 0, t0 = 0; i < slots.size(); t0 += counts[i], ++i) toks[i] = tk.data() + t0;
            std::vector<int> meta(MetaView::ints(e->maxT, S), 0);
            REQUIRE(e->fill_meta(meta.data(), slots, counts, toks, outmode, &R) == T, B200RWKV_ERR_INVALID, "internal: step metadata");
            metas.push_back((int*)up(meta.data(), meta.size() * 4));
            if (l == 0) meta0 = meta;
        }
        e->d_meta = metas[0];
        sh = e->step_shape(T, R);
    }
    // Snapshot tokens tok[k] with records rec + k * ld (the caller checked them with snap_args_ok): the step's snapshot block
    // from the engine's fill_snap, uploaded, and the step's shape as infer sets it.  Returns the device copy of the records;
    // the block's record table is snap_table.
    float* snap_start(int nsnap, const int32_t* tok, const float* rec, int64_t ld) {
        e->meta_ints = MetaView::ints(e->maxT, S);
        e->snap_sizes();
        float* d_rec = (float*)up(rec, (size_t)nsnap * ld * 4);
        std::vector<b200rwkv_engine::SnapTok> tk;
        for (int k = 0; k < nsnap; ++k) tk.push_back({tok[k], d_rec + (size_t)k * ld, nullptr});
        std::vector<uint8_t> hs(e->snap_bytes);
        const int X = e->fill_snap(hs.data(), meta0.data(), T, tk);
        uint8_t* d = (uint8_t*)up(hs.data(), hs.size());
        snap_meta = MetaView{reinterpret_cast<const int*>(d), e->maxT, S};
        snap_table = reinterpret_cast<float* const*>(d + e->snap_meta_bytes);
        sh.snap = true;
        sh.MTX = X > 0 ? mt_bucket(X) : 0;
        return d_rec;
    }
    // the layout start() built the blocks with, whatever the entry sets e->maxT to afterwards
    MetaView meta(int l) const { return MetaView{metas[l], A16_MAX_ROWS, S}; }
    void* up(const void* h, size_t bytes) {
        void* d = e->dalloc(bytes, false);
        CK(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice));
        return d;
    }
    // per-token rows as the engine's activation buffers hold them: sh.rows rows, the ones past T filled with NaN so that a read
    // outside the step shows in the output
    float* rows_up(const float* h, int cols) {
        if (!h) return nullptr;
        float* d = (float*)e->dalloc((size_t)sh.rows * cols * 4, false);
        CK(cudaMemset(d, 0xFF, (size_t)sh.rows * cols * 4));
        CK(cudaMemcpy(d, h, (size_t)T * cols * 4, cudaMemcpyHostToDevice));
        return d;
    }
};

// Operator-level entry for the parity tests: ONE WKV launch of a step (recurrence + GroupNorm + bonus + gate) on caller-supplied
// head vectors and state pool, no model around it.  The step comes from OpStep, the launch from launch_wkv (kernel per version
// and output form, grid, shared memory, programmatic dependent launch), the k-major decay slice from wd2_k_major and the d1
// operand from the f16 conversion of the projection operands: a step runs exactly this.  The committed fla fixtures
// (tests/golden/wkv6_fla.npz, wkv7_fla.npz) and the float64 reference of tests/test_gpu_wkv.py reach the CUDA kernels through it.
int32_t b200rwkv_op_wkv(int32_t device, const b200rwkv_wkv_args* args) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(args, B200RWKV_ERR_INVALID, "null arguments");
    const b200rwkv_wkv_args& x = *args;
    const int version = x.version;
    REQUIRE(version == 5 || version == 6 || version == 7, B200RWKV_ERR_UNSUPPORTED, "version must be 5, 6 or 7");
    REQUIRE(x.H >= 1 && x.H <= 128, B200RWKV_ERR_INVALID, "H must be 1..128 (num_emb <= 8192)");
    OpStep st(x.S, x.nslot, x.slot, x.count, x.precision);
    REQUIRE(x.r && x.k && x.v && x.g && x.lnx_w && x.lnx_b && x.state && x.out, B200RWKV_ERR_INVALID, "null r, k, v, g, ln_x, state or out");
    const bool fold = version == 6 && (x.d1 || x.time_decay_w2 || x.decay_bias);
    if (fold) {
        REQUIRE(x.d1 && x.time_decay_w2 && x.decay_bias, B200RWKV_ERR_INVALID, "the decay fold needs d1, time_decay_w2 and decay_bias");
        REQUIRE(x.Dd >= 8 && x.Dd <= 128 && x.Dd % 8 == 0, B200RWKV_ERR_UNSUPPORTED, "the decay fold needs Dd <= 128 and Dd % 8 == 0");
    }
    if (version == 5) REQUIRE(x.w && x.u, B200RWKV_ERR_INVALID, "v5 needs w (static) and u");
    if (version == 6) REQUIRE((x.w || fold) && x.u, B200RWKV_ERR_INVALID, "v6 needs u and w or the decay fold");
    if (version == 7) {
        REQUIRE(x.w && x.a && x.k_k && x.k_a && x.r_k && x.v_first, B200RWKV_ERR_INVALID, "v7 needs w, a, k_k, k_a, r_k and v_first");
        REQUIRE(x.layer0 || x.nu, B200RWKV_ERR_INVALID, "v7 layers after 0 need nu");
    }

    snap_args_ok(x.nsnap, x.snap_tok, x.snap_rec, x.snap_ld, x.snap_off, (int64_t)x.H * 64 * 64, st.T);

    const int H = x.H, S = x.S, Cc = H * 64, T = st.T;
    st.start(device, 1, nullptr, std::vector<int>(x.nslot, 0));
    float* d_rec = x.nsnap > 0 ? st.snap_start(x.nsnap, x.snap_tok, x.snap_rec, x.snap_ld) : nullptr;
    const StepShape& sh = st.sh;
    wkv_smem_limits();

    auto rows_up = [&](const float* h) { return st.rows_up(h, Cc); };
    auto vec_up = [&](const float* h) { return h ? (const float*)st.up(h, (size_t)Cc * 4) : nullptr; };
    WkvParams p;
    memset(&p, 0, sizeof(p));
    p.version = version; p.ld = Cc; p.meta = st.meta(0); p.H = H;
    p.snap_rec = st.snap_table; p.snap_off = (size_t)x.snap_off;
    const size_t state_bytes = (size_t)S * H * 64 * 64 * 4;
    p.state = (float*)st.up(x.state, state_bytes);
    p.r = rows_up(x.r); p.k = rows_up(x.k); p.v = rows_up(x.v); p.g = rows_up(x.g);
    if (version == 5) p.w_static = vec_up(x.w);
    else if (!fold) p.w = rows_up(x.w);
    p.u = version != 7 ? vec_up(x.u) : nullptr;
    p.lnx_w = vec_up(x.lnx_w); p.lnx_b = vec_up(x.lnx_b);
    if (version == 7) {
        p.a = rows_up(x.a); p.nu = x.layer0 ? nullptr : rows_up(x.nu);
        p.v_first = rows_up(x.v_first); p.layer0 = x.layer0 != 0;
        p.k_k = vec_up(x.k_k); p.k_a = vec_up(x.k_a); p.r_k = vec_up(x.r_k);
    }
    if (fold) {
        const std::vector<__half> wt = wd2_k_major(reinterpret_cast<const __half*>(x.time_decay_w2), 0, H, x.Dd);
        p.wd2t = (const __half*)st.up(wt.data(), wt.size() * 2);
        p.decay_bias = vec_up(x.decay_bias);
        p.Dd = x.Dd;
        float* d1 = (float*)st.up(x.d1, (size_t)T * x.Dd * 4);
        __half* a16 = (__half*)st.e->dalloc(a16_halves(x.Dd) * 2, true);
        a16_from_f32_kernel<<<cdiv(T * x.Dd, 256), 256>>>(d1, T, x.Dd, sh.th, sh.split, a16);
        CK(cudaGetLastError());
        p.d1 = a16;
    }
    // the output in the A16 layout of `th` token rows, the caller's contents first
    std::vector<uint16_t> h16 = a16_pack(x.out, Cc, Cc, sh.th, 0, Cc);
    p.out = (__half*)st.up(h16.data(), h16.size() * 2);
    CK(cudaDeviceSynchronize());                   // every upload has landed before the launch
    st.e->launch_wkv(p, sh, st.e->stream, nullptr);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st.e->stream));
    CK(cudaMemcpy(h16.data(), p.out, h16.size() * 2, cudaMemcpyDeviceToHost));
    a16_unpack(h16, Cc, Cc, sh.th, sh.th, 0, Cc, x.out);
    CK(cudaMemcpy(x.state, p.state, state_bytes, cudaMemcpyDeviceToHost));
    if (version == 7) CK(cudaMemcpy(x.v_first, p.v_first, (size_t)T * Cc * 4, cudaMemcpyDeviceToHost));
    if (d_rec) CK(cudaMemcpy(x.snap_rec, d_rec, (size_t)x.nsnap * x.snap_ld * 4, cudaMemcpyDeviceToHost));
    API_END
}

// Operator-level entry for the parity tests: ONE LN stage of a step (embed + LN0, LN1 / LN2, the RWKV-6 front half or ln_out)
// on caller-supplied rows and pool, no model.  The step comes from OpStep, the parameter blocks are the kernels' own, and the
// launch from launch_embed / launch_ln / launch_pre6 / launch_ln_out (kernel choice, cluster and programmatic-dependent-launch
// attributes, token rows of the operands): a step runs exactly this.  tests/test_gpu_ln.py holds the LN kernels to a float64
// reference through it.
int32_t b200rwkv_op_ln(int32_t device, const b200rwkv_ln_args* args) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(args, B200RWKV_ERR_INVALID, "null arguments");
    const b200rwkv_ln_args& x = *args;
    const int stage = x.stage, C = x.C, S = x.S, NL = x.launches;
    REQUIRE(stage >= 0 && stage <= 3, B200RWKV_ERR_INVALID, "stage must be 0 (embed), 1 (LN), 2 (front half) or 3 (ln_out)");
    REQUIRE(C >= 64 && C <= LN_MAXC && C % 64 == 0, B200RWKV_ERR_INVALID, "C must be a multiple of 64 and <= 8192");
    REQUIRE(NL >= 1 && NL <= 16, B200RWKV_ERR_INVALID, "launches must be 1..16");
    REQUIRE(x.batch_invariant == 0 || x.batch_invariant == 1, B200RWKV_ERR_INVALID, "batch_invariant must be 0 or 1");
    OpStep st(S, x.nslot, x.slot, x.count, x.precision);
    const int T = st.T;
    if (stage == 0) {
        REQUIRE(x.emb && x.V >= 1 && x.tokens && x.ln_w && x.ln_b && x.x_out, B200RWKV_ERR_INVALID,
                "embed needs emb, V >= 1, tokens, ln_w, ln_b and x_out");
        for (size_t i = 0; i < (size_t)NL * T; ++i)
            REQUIRE(x.tokens[i] < (uint32_t)x.V, B200RWKV_ERR_INVALID, "token id " + std::to_string(x.tokens[i]) + " is outside the vocabulary");
    } else {
        REQUIRE(x.x_in && x.ln_w && x.ln_b, B200RWKV_ERR_INVALID, "null x_in, ln_w or ln_b");
        REQUIRE(x.n_parts >= 0 && x.n_parts <= 8 && x.n_gate >= 0 && x.n_gate <= 8, B200RWKV_ERR_INVALID, "n_parts and n_gate must be 0..8");
        REQUIRE(x.n_parts == 0 || x.parts, B200RWKV_ERR_INVALID, "null parts");
        REQUIRE(x.n_gate == 0 || x.gates, B200RWKV_ERR_INVALID, "null gates");
        REQUIRE(x.n_gate == 0 || (C % x.n_gate == 0 && (C / x.n_gate) % 4 == 0), B200RWKV_ERR_INVALID,
                "gate blocks (C / n_gate columns) must be whole multiples of 4 columns");
        REQUIRE(!x.commit_src == !x.commit_dst, B200RWKV_ERR_INVALID, "the commit needs both commit_src and commit_dst");
    }
    if (stage == 1 || stage == 2) {
        REQUIRE(x.n_mix >= 1 && x.n_mix <= 6, B200RWKV_ERR_INVALID, "n_mix must be 1..6");
        REQUIRE(x.shift_state && x.mu && x.mix_out && x.xx_out, B200RWKV_ERR_INVALID, "null shift_state, mu, mix_out or xx_out");
        REQUIRE(x.x_out || x.n_parts == 0, B200RWKV_ERR_INVALID, "in place (x_out NULL) takes no parts");
    }
    if (stage == 2) {
        REQUIRE((T <= 16 || x.batch_invariant) && pre6_fits(x.Dm, C), B200RWKV_ERR_UNSUPPORTED,
                "the front half runs decode-shaped steps (T <= 16; up to 128 with batch_invariant) with Dm 32 or 64, C % 128 == 0 "
                "and C <= 4096");
        REQUIRE(x.n_mix == 1 && x.sx_out && x.W1 && x.W2 && x.mu5 && x.lora_out && x.out5, B200RWKV_ERR_INVALID,
                "the front half needs n_mix 1, sx_out, W1, W2, mu5, lora_out and out5");
    }
    std::vector<int> outmode(x.nslot, 0);
    if (stage == 3) {
        REQUIRE(x.option && x.head_out, B200RWKV_ERR_INVALID, "ln_out needs option and head_out");
        for (int i = 0; i < x.nslot; ++i) {
            REQUIRE(x.option[i] >= B200RWKV_OPTION_LAST && x.option[i] <= B200RWKV_OPTION_NONE, B200RWKV_ERR_INVALID, "bad option");
            outmode[i] = x.option[i] == B200RWKV_OPTION_FULL ? 2 : (x.option[i] == B200RWKV_OPTION_LAST ? 1 : 0);
        }
    }
    snap_args_ok(x.nsnap, x.snap_tok, x.snap_rec, x.snap_ld, x.snap_off, C, T);
    if (x.nsnap > 0) {
        REQUIRE(stage != 0, B200RWKV_ERR_INVALID, "the embed stage takes no snapshots");
        REQUIRE(NL == 1, B200RWKV_ERR_INVALID, "snapshots take one launch");
        // a step's ln_out always commits the last layer's channel-mix shift, and its kernel copies commit_src unchecked
        REQUIRE(stage != 3 || (x.commit_src && x.snap_head_out), B200RWKV_ERR_INVALID, "ln_out snapshots need the commit and snap_head_out");
    }

    st.start(device, NL, x.tokens, outmode);
    float* d_rec = x.nsnap > 0 ? st.snap_start(x.nsnap, x.snap_tok, x.snap_rec, x.snap_ld) : nullptr;
    b200rwkv_engine* e = st.e.get();
    e->ln_cluster_ok = ln_cluster_fits(C);         // as build() decides it for a model of C channels
    e->batch_inv = x.batch_invariant != 0;
    const StepShape& sh = st.sh;
    const int th = sh.th;
    const int hrows = std::max(sh.th_rows, 16);    // the caller's head_out has 16 rows even when the step has no output row
    const int xrows = sh.split ? 32 : 16 * sh.MTX;  // snap_head_out

    auto rows_down = [&](float* h, const float* d) { CK(cudaMemcpy(h, d, (size_t)T * C * 4, cudaMemcpyDeviceToHost)); };
    // A16 operands: `nmat` matrices of K columns with `tr` token rows, exchanged with the caller as [nmat][tr][K]
    auto a16_up = [&](const uint16_t* h, int nmat, int K, int tr) {
        const std::vector<uint16_t> b = a16_pack(h, nmat * K, K, tr, (size_t)tr * K, K);
        return (__half*)st.up(b.data(), b.size() * 2);
    };
    auto a16_down = [&](uint16_t* h, const __half* d, int nmat, int K, int tr) {
        std::vector<uint16_t> b(a16_halves(K) * nmat);
        CK(cudaMemcpy(b.data(), d, b.size() * 2, cudaMemcpyDeviceToHost));
        a16_unpack(b, nmat * K, K, tr, tr, (size_t)tr * K, K, h);
    };

    const size_t TC = (size_t)T * C;
    const float* ln_w = (const float*)st.up(x.ln_w, (size_t)C * 4);
    const float* ln_b = (const float*)st.up(x.ln_b, (size_t)C * 4);
    float* cdst = x.commit_dst ? (float*)st.up(x.commit_dst, (size_t)S * C * 4) : nullptr;
    unsigned* gbar = (unsigned*)e->dalloc(256, true);      // the front half's barrier counters, shared by every launch
    float** hid_tab = nullptr;
    std::vector<float*> hid_rows(NL, nullptr);
    const int gcl = x.n_gate > 0 ? C / x.n_gate : 0;
    auto residual = [&](auto& p, int l) {          // LnMixParams / LnOutParams: x_in + gate (.) sum parts of launch l
        p.x_in = st.rows_up(x.x_in + l * TC, C);
        p.C = C;
        p.meta = st.meta(l);
        p.n_parts = x.n_parts;
        for (int q = 0; q < x.n_parts; ++q) p.parts[q] = st.rows_up(x.parts + ((size_t)l * x.n_parts + q) * TC, C);
        p.n_gate = x.n_gate;
        p.gate_cl = gcl;
        for (int q = 0; q < x.n_gate; ++q) p.gates[q] = st.rows_up(x.gates + ((size_t)l * x.n_gate + q) * T * gcl, gcl);
        p.ln_w = ln_w; p.ln_b = ln_b;
        p.commit_dst = cdst;
        p.commit_src = x.commit_src ? st.rows_up(x.commit_src + l * TC, C) : nullptr;
        if (x.hidden) hid_rows[l] = st.rows_up(x.hidden + l * TC, C);
    };

    std::vector<EmbedParams> em(NL);
    std::vector<LnMixParams> lm(NL);
    std::vector<Pre6Params> pq(NL);
    std::vector<LnOutParams> lo(NL);
    if (stage == 0) {
        const __half* emb = (const __half*)st.up(x.emb, (size_t)x.V * C * 2);
        for (int l = 0; l < NL; ++l) {
            EmbedParams& p = em[l];
            memset(&p, 0, sizeof(p));
            p.emb = emb; p.C = C; p.V = x.V; p.meta = st.meta(l);
            p.ln_w = ln_w; p.ln_b = ln_b;
            p.x_out = st.rows_up(x.x_out + l * TC, C);
        }
    } else if (stage == 1 || stage == 2) {
        const float* shift = (const float*)st.up(x.shift_state, (size_t)S * C * 4);
        const float* mu = (const float*)st.up(x.mu, (size_t)x.n_mix * C * 4);
        if (x.hidden) hid_tab = (float**)e->dalloc((size_t)NL * sizeof(float*), true);
        for (int l = 0; l < NL; ++l) {
            LnMixParams& p = lm[l];
            memset(&p, 0, sizeof(p));
            residual(p, l);
            p.x_out = x.x_out ? st.rows_up(x.x_out + l * TC, C) : const_cast<float*>(p.x_in);
            p.shift_state = shift;
            p.n_mix = x.n_mix;
            const __half* mix = a16_up(x.mix_out + (size_t)l * x.n_mix * th * C, x.n_mix, C, th);
            for (int j = 0; j < x.n_mix; ++j) { p.mu[j] = mu + (size_t)j * C; p.mix_out[j] = const_cast<__half*>(mix) + j * a16_halves(C); }
            p.xx_out = st.rows_up(x.xx_out + l * TC, C);
            p.sx_out = x.sx_out ? st.rows_up(x.sx_out + l * TC, C) : nullptr;
            p.hid_slot = hid_tab ? hid_tab + l : nullptr;
            p.snap_rec = st.snap_table; p.snap_off = (size_t)x.snap_off;
        }
        if (hid_tab) CK(cudaMemcpy(hid_tab, hid_rows.data(), (size_t)NL * sizeof(float*), cudaMemcpyHostToDevice));
        if (stage == 2) {
            const int Dm = x.Dm;
            const __half* W1 = (const __half*)st.up(x.W1, (size_t)5 * Dm * C * 2);
            const __half* W2 = (const __half*)st.up(x.W2, (size_t)5 * C * Dm * 2);
            const float* mu5 = (const float*)st.up(x.mu5, (size_t)5 * C * 4);
            for (int l = 0; l < NL; ++l) {
                Pre6Params& q = pq[l];
                memset(&q, 0, sizeof(q));
                q.ln = lm[l];
                q.W1 = W1; q.W2 = W2;
                const __half* o5 = a16_up(x.out5 + (size_t)l * 5 * th * C, 5, C, th);
                for (int j = 0; j < 5; ++j) { q.mu[j] = mu5 + (size_t)j * C; q.out[j] = const_cast<__half*>(o5) + j * a16_halves(C); }
                q.lora = const_cast<__half*>(a16_up(x.lora_out + (size_t)l * 5 * th * Dm, 5, Dm, th));
                q.lora_stride = (int)a16_halves(Dm);
                q.Dm = Dm;
                q.gbar = gbar;
            }
        }
    } else {
        for (int l = 0; l < NL; ++l) {
            LnOutParams& p = lo[l];
            memset(&p, 0, sizeof(p));
            residual(p, l);
            p.head_in = const_cast<__half*>(a16_up(x.head_out + (size_t)l * hrows * C, 1, C, hrows));
            p.hidden_out = hid_rows[l];
            p.snap_rec = st.snap_table; p.snap_off = (size_t)x.snap_off;
            if (sh.MTX > 0) {
                p.snap_meta = st.snap_meta;
                p.snap_head_in = const_cast<__half*>(a16_up(x.snap_head_out, 1, C, xrows));
            }
        }
    }
    CK(cudaDeviceSynchronize());                   // every upload has landed before the launches
    LnPick pick{};
    for (int l = 0; l < NL; ++l) {
        if (stage == 0) pick = e->launch_embed(em[l], sh, e->stream, nullptr);
        else if (stage == 1) pick = e->launch_ln(lm[l], sh, e->stream, nullptr);
        else if (stage == 2) {
            if (sh.MT > 1) e->launch_ln(pq[l].ln, sh, e->stream, nullptr);     // as enqueue_step runs a longer step's LN1
            pick = e->launch_pre6(pq[l], sh, e->stream, nullptr);
        }
        else pick = e->launch_ln_out(lo[l], sh, e->stream, nullptr);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    for (int l = 0; l < NL; ++l) {
        if (stage == 0) { rows_down(x.x_out + l * TC, em[l].x_out); continue; }
        if (x.hidden) rows_down(x.hidden + l * TC, hid_rows[l]);
        if (stage == 3) {
            a16_down(x.head_out + (size_t)l * hrows * C, lo[l].head_in, 1, C, hrows);
            if (lo[l].snap_head_in) a16_down(x.snap_head_out, lo[l].snap_head_in, 1, C, xrows);
            continue;
        }
        const LnMixParams& p = lm[l];
        if (x.x_out) rows_down(x.x_out + l * TC, p.x_out);
        else rows_down(x.x_in + l * TC, p.x_in);
        rows_down(x.xx_out + l * TC, p.xx_out);
        if (x.sx_out) rows_down(x.sx_out + l * TC, p.sx_out);
        a16_down(x.mix_out + (size_t)l * x.n_mix * th * C, p.mix_out[0], x.n_mix, C, th);
        if (stage == 2) {
            a16_down(x.out5 + (size_t)l * 5 * th * C, pq[l].out[0], 5, C, th);
            a16_down(x.lora_out + (size_t)l * 5 * th * x.Dm, pq[l].lora, 5, x.Dm, th);
        }
    }
    if (cdst) CK(cudaMemcpy(x.commit_dst, cdst, (size_t)S * C * 4, cudaMemcpyDeviceToHost));
    if (d_rec) CK(cudaMemcpy(x.snap_rec, d_rec, (size_t)x.nsnap * x.snap_ld * 4, cudaMemcpyDeviceToHost));
    if (x.kernel_out) { x.kernel_out[0] = pick.kernel; x.kernel_out[1] = pick.variant; x.kernel_out[2] = pick.split; }
    API_END
}

// Operator-level entry for the parity tests: ONE projection plan built by the engine's own planner (make_launch: grid choice,
// stream-K cuts, workspace slots, repacking or quantisation) over caller-supplied matrices, launched by launch_gemm (kernel
// per token-tile count, ring size, split operands, programmatic dependent launch) `launches` times back to back, as the
// engine reuses a plan step after step.  A temporary engine object carries just what those two need.
// ntail > 0 (b200rwkv_op_gemm_tail): segment 0 is a W' plan with ntail adapter tail blocks, built through make_launch's own
// tail path from one stand-in adapter file per block (lora.1 = that block's columns, alpha 1), and its operand's tail blocks
// hold tail_u as the shrink kernel would have written them.
static int32_t op_gemm_run(int32_t device, int32_t T, int32_t precision, int32_t quant_type, int32_t grid, int32_t launches,
                           int32_t nseg, const b200rwkv_gemm_seg* seg, int32_t* plan_out, int32_t ntail = 0,
                           const uint16_t* tail_e = nullptr, const uint16_t* tail_u = nullptr) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(seg && nseg >= 1 && nseg <= GEMM_MAX_SEG, B200RWKV_ERR_INVALID, "nseg must be 1..8");
    REQUIRE(T >= 1 && T <= A16_MAX_ROWS, B200RWKV_ERR_INVALID, "T must be 1..128");
    REQUIRE(precision == 0 || precision == 1, B200RWKV_ERR_INVALID, "precision must be 0 or 1");
    REQUIRE(grid >= 0 && launches >= 1 && launches <= 16, B200RWKV_ERR_INVALID, "grid must be >= 0 and launches 1..16");
    REQUIRE(quant_type == QT_NONE || quant_type == QT_INT8 || quant_type == QT_NF4 || quant_type == QT_FP8 || quant_type == QT_INT4,
            B200RWKV_ERR_UNSUPPORTED, "quant_type must be 0, 1, 2, 4 or 6");
    REQUIRE(precision == 0 || (T <= 16 && quant_type == QT_NONE), B200RWKV_ERR_UNSUPPORTED,
            "precision 1 runs decode-shaped steps (T <= 16) over f16 weights");
    for (int i = 0; i < nseg; ++i) {
        const b200rwkv_gemm_seg& s = seg[i];
        const std::string tag = "segment " + std::to_string(i) + ": ";
        REQUIRE(s.N >= 1 && s.K >= 1 && (int64_t)s.N * s.K <= ((int64_t)1 << 31) && s.w && s.x && s.out, B200RWKV_ERR_INVALID,
                tag + "bad N / K or a null matrix");
        REQUIRE(s.act >= ACT_NONE && s.act <= ACT_V7DECAY && s.out_mode >= OUT_F32 && s.out_mode <= OUT_LERP_A16 && s.grp >= 0,
                B200RWKV_ERR_INVALID, tag + "bad act / out_mode / grp");
        REQUIRE(s.ldo >= s.N && s.ldo <= (1 << 24), B200RWKV_ERR_INVALID, tag + "ldo must be >= N");
        REQUIRE(s.out_mode != OUT_LERP_A16 || (s.lerp_xx && s.lerp_sx && s.lerp_mu), B200RWKV_ERR_INVALID, tag + "ddlerp needs xx, sx and mu");
        REQUIRE(s.out_mode == OUT_F32 || (s.N % 8 == 0 && s.grp % 8 == 0), B200RWKV_ERR_UNSUPPORTED,
                tag + "f16 outputs are written in chunks of 8 columns: N and grp must be multiples of 8");
        REQUIRE(quant_type == QT_NONE || s.K % GEMM_BK == 0, B200RWKV_ERR_UNSUPPORTED, tag + "quantised matrices need K % 128 == 0");
    }
    // one entry of T tokens: make_launch points every launch's valid token rows at the step metadata's T
    const int32_t slot0 = 0;
    OpStep st(1, 1, &slot0, &T, precision);
    st.start(device, 1, nullptr, {0});
    b200rwkv_engine* e = st.e.get();
    const StepShape& sh = st.sh;
    const int th = sh.th;                          // token rows of every operand / output in the A16 layout, rows of `out`
    CK(cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, device));
    e->maxT = th;                                  // sizes the stream-K workspace (make_launch); the metadata keeps its layout
    gemm_smem_limits(quant_type);
    // f16 destination in the A16 layout: `grp` columns per matrix (one matrix of ldo columns without groups)
    auto mat_cols = [](const b200rwkv_gemm_seg& s) { return s.grp > 0 ? s.grp : s.ldo; };
    std::vector<StTensor> wt(nseg);
    std::vector<SegDesc> sv(nseg);
    for (int i = 0; i < nseg; ++i) {
        const b200rwkv_gemm_seg& s = seg[i];
        wt[i].name = "op_gemm." + std::to_string(i) + ".weight";
        wt[i].dtype = "F16";
        wt[i].shape = {s.N, s.K};
        wt[i].data = reinterpret_cast<const uint8_t*>(s.w);
        wt[i].nbytes = (size_t)s.N * s.K * 2;
        SegDesc& d = sv[i];
        d.t = &wt[i]; d.N = s.N; d.K = s.K;
        d.proto.out_mode = s.out_mode; d.proto.act = s.act; d.proto.grp = s.out_mode == OUT_F32 ? 0 : s.grp;
        d.proto.bias = s.bias ? (const float*)st.up(s.bias, (size_t)s.N * 4) : nullptr;
        if (s.out_mode == OUT_LERP_A16) { d.proto.aux2 = (const float*)st.up(s.lerp_mu, (size_t)s.N * 4); d.proto.ld_aux = s.N; }
        if (s.out_mode != OUT_F32) d.proto.grp_stride = (int)a16_halves(mat_cols(s));
        else d.proto.ldo = s.ldo;
    }
    std::vector<StFile> tail_files(ntail);
    std::vector<std::vector<uint16_t>> tail_cols(ntail);
    for (int a = 0; a < ntail; ++a) {
        const int N = seg[0].N;
        tail_cols[a].resize((size_t)N * GEMM_BK);
        for (int n = 0; n < N; ++n)
            memcpy(&tail_cols[a][(size_t)n * GEMM_BK], tail_e + ((size_t)n * ntail + a) * GEMM_BK, GEMM_BK * 2);
        StTensor& t = tail_files[a].tensors["op_gemm.0.lora.1"];
        t.name = "op_gemm.0.lora.1";
        t.dtype = "F16";
        t.shape = {N, GEMM_BK};
        t.data = reinterpret_cast<const uint8_t*>(tail_cols[a].data());
        t.nbytes = tail_cols[a].size() * 2;
        e->adapters.push_back({&tail_files[a], 1.f});
    }
    sv[0].ad_tail = ntail;
    GemmLaunch g = e->make_launch(sv, grid, quant_type);
    {
        std::vector<b200rwkv_engine::WeightIn> in;      // the weight fills the plan recorded, as the build runs them
        for (const StTensor& t : wt) in.push_back({t.name, &t, nullptr, B200RWKV_DTYPE_F16, t.numel()});
        CK(cudaDeviceSynchronize());
        e->fill_weights(in);
    }
    e->gemm_ws = (float*)e->dalloc(e->gemm_ws_floats * 4, false);
    g.p.ws = e->gemm_ws;

    // the plan as launch_gemm will run it, and the cut of every tile by the kernel's own formula
    const int G = sh.MT >= 4 ? g.grid_wide : g.grid;
    const unsigned TB = (unsigned)g.p.total_blocks;
    int maxc = 0;
    for (int i = 0; i < nseg; ++i) {
        const GemmSeg& sg = g.p.seg[i];
        for (int t = 0; t < sg.tiles; ++t) {
            const unsigned tb0 = (unsigned)(sg.blk_begin + t * sg.KB);
            const int c_first = (int)(((unsigned long long)(tb0 + 1) * (unsigned)G - 1) / TB);
            const int c_last = (int)(((unsigned long long)(tb0 + sg.KB) * (unsigned)G - 1) / TB);
            maxc = std::max(maxc, c_last - c_first + 1);
        }
    }
    REQUIRE(maxc <= g.p.max_contrib, B200RWKV_ERR_INVALID, "internal: a tile has more contributors than workspace slots");
    if (plan_out) { plan_out[0] = G; plan_out[1] = g.p.total_blocks; plan_out[2] = g.total_tiles; plan_out[3] = maxc; }

    // operands and outputs of every launch; the caller's output contents go up first
    std::vector<GemmLaunch> runs(launches, g);
    std::vector<std::vector<uint16_t>> h16(nseg);         // f16 bits of an A16 destination
    Buf<float> xs((size_t)T * std::max_element(seg, seg + nseg, [](const b200rwkv_gemm_seg& a, const b200rwkv_gemm_seg& b) { return a.K < b.K; })->K * 4);
    for (int l = 0; l < launches; ++l) {
        for (int i = 0; i < nseg; ++i) {
            const b200rwkv_gemm_seg& s = seg[i];
            GemmSeg& sg = runs[l].p.seg[i];
            const int nt = i == 0 ? ntail : 0;
            __half* a = (__half*)e->dalloc((a16_halves(s.K) + (size_t)nt * A16_KB_HALVES) * 2, true);
            CK(cudaMemcpy(xs, s.x + (size_t)l * T * s.K, (size_t)T * s.K * 4, cudaMemcpyHostToDevice));
            a16_from_f32_kernel<<<(int)std::min<size_t>(((size_t)T * s.K + 255) / 256, (size_t)e->num_sms * 8), 256>>>(xs, T, s.K, th, sh.split, a);
            CK(cudaGetLastError());
            CK(cudaDeviceSynchronize());           // xs is refilled by the next upload
            if (nt) {                              // the operand's tail blocks after its own k blocks, as the shrink writes them
                std::vector<uint16_t> u((size_t)nt * A16_KB_HALVES, 0);
                for (int t = 0; t < T; ++t)
                    for (int k = 0; k < nt * GEMM_BK; ++k) u[a16_index(t, k, th)] = tail_u[(size_t)t * nt * GEMM_BK + k];
                CK(cudaMemcpy(a + a16_halves(s.K), u.data(), u.size() * 2, cudaMemcpyHostToDevice));
            }
            sg.A = a;
            const size_t cells = (size_t)th * s.ldo;
            if (s.out_mode == OUT_F32) {
                sg.out = st.up((const float*)s.out + l * cells, cells * 4);
                continue;
            }
            std::vector<uint16_t>& h = h16[i];
            h = a16_pack((const uint16_t*)s.out + l * cells, s.ldo, mat_cols(s), th, mat_cols(s), s.ldo);
            sg.out = st.up(h.data(), h.size() * 2);
            if (s.out_mode == OUT_LERP_A16) {          // all `th` rows exist, as in the engine's activation buffers
                float* xx = (float*)e->dalloc((size_t)th * s.N * 4, true);
                float* sx = (float*)e->dalloc((size_t)th * s.N * 4, true);
                CK(cudaMemcpy(xx, s.lerp_xx + (size_t)l * T * s.N, (size_t)T * s.N * 4, cudaMemcpyHostToDevice));
                CK(cudaMemcpy(sx, s.lerp_sx + (size_t)l * T * s.N, (size_t)T * s.N * 4, cudaMemcpyHostToDevice));
                sg.aux0 = xx;
                sg.aux1 = sx;
            }
        }
    }
    CK(cudaDeviceSynchronize());                   // every upload has landed before the projection stream starts
    for (const GemmLaunch& r : runs) e->launch_gemm(r, sh, e->stream, nullptr);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    for (int l = 0; l < launches; ++l)
        for (int i = 0; i < nseg; ++i) {
            const b200rwkv_gemm_seg& s = seg[i];
            const size_t cells = (size_t)th * s.ldo;
            if (s.out_mode == OUT_F32) {
                CK(cudaMemcpy((float*)s.out + l * cells, runs[l].p.seg[i].out, cells * 4, cudaMemcpyDeviceToHost));
                continue;
            }
            std::vector<uint16_t>& h = h16[i];
            CK(cudaMemcpy(h.data(), runs[l].p.seg[i].out, h.size() * 2, cudaMemcpyDeviceToHost));
            a16_unpack(h, s.ldo, mat_cols(s), th, th, mat_cols(s), s.ldo, (uint16_t*)s.out + l * cells);
        }
    API_END
}

int32_t b200rwkv_op_gemm(int32_t device, int32_t T, int32_t precision, int32_t quant_type, int32_t grid, int32_t launches,
                         int32_t nseg, const b200rwkv_gemm_seg* seg, int32_t* plan_out) {
    return op_gemm_run(device, T, precision, quant_type, grid, launches, nseg, seg, plan_out);
}

// Operator-level entry for the parity tests: one W' launch (b200rwkv_op_gemm's planner and launcher, adapter tails)
int32_t b200rwkv_op_gemm_tail(int32_t device, int32_t T, int32_t quant_type, int32_t grid, int32_t n, const b200rwkv_gemm_seg* seg,
                              const uint16_t* tail_e, const uint16_t* tail_u, int32_t* plan_out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(n >= 1 && n <= AD_MAX, B200RWKV_ERR_INVALID, "n must be 1..8");
    REQUIRE(seg && tail_e && tail_u, B200RWKV_ERR_INVALID, "null segment or tail");
    return op_gemm_run(device, T, 0, quant_type, grid, 1, 1, seg, plan_out, n, tail_e, tail_u);
    API_END
}

// Operator-level entry for the parity tests: the kept-row gather after a step (keep_rows_kernel) over caller-supplied vocabulary
// shards, no model.  The step's metadata comes from OpStep, every shard sits in its own allocation as each rank's logits block
// does, and the launch is enqueue_keep's: what rank 0 of a `world`-rank engine runs after a step of these entries.
int32_t b200rwkv_op_keep(int32_t device, const b200rwkv_keep_args* args) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(args, B200RWKV_ERR_INVALID, "null arguments");
    const b200rwkv_keep_args& x = *args;
    REQUIRE(x.world >= 1 && x.world <= 8, B200RWKV_ERR_INVALID, "world must be 1..8");
    REQUIRE(x.Vl >= 1 && (int64_t)x.Vl * x.world <= ((int64_t)1 << 22), B200RWKV_ERR_INVALID, "Vl must be >= 1 with world * Vl <= 4194304");
    OpStep st(x.S, x.nslot, x.slot, x.count, 0);
    REQUIRE(x.option && x.keep, B200RWKV_ERR_INVALID, "null option or keep");
    std::vector<int> outmode(x.nslot, 0);
    int R = 0;
    for (int i = 0; i < x.nslot; ++i) {
        REQUIRE(x.option[i] >= B200RWKV_OPTION_LAST && x.option[i] <= B200RWKV_OPTION_NONE, B200RWKV_ERR_INVALID, "bad option");
        outmode[i] = x.option[i] == B200RWKV_OPTION_FULL ? 2 : (x.option[i] == B200RWKV_OPTION_LAST ? 1 : 0);
        R += x.option[i] == B200RWKV_OPTION_FULL ? x.count[i] : (x.option[i] == B200RWKV_OPTION_LAST ? 1 : 0);
    }
    REQUIRE(R == 0 || x.shards, B200RWKV_ERR_INVALID, "null shards");
    const int world = x.world, Vl = x.Vl, V = world * Vl;
    const size_t keep_bytes = (size_t)x.S * V * 4;
    st.start(device, 1, nullptr, outmode);
    b200rwkv_engine* e = st.e.get();
    e->rank = 0; e->world = world; e->Vl = Vl; e->V = V;
    e->d_keep = (float*)st.up(x.keep, keep_bytes);
    e->off_logits = 0;
    for (int q = 0; q < world; ++q) e->peer_base[q] = (uint8_t*)st.up(x.shards + (size_t)q * R * Vl, (size_t)R * Vl * 4);
    CK(cudaDeviceSynchronize());                   // every upload has landed before the launch
    e->enqueue_keep(e->stream, st.sh.MTR);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(x.keep, e->d_keep, keep_bytes, cudaMemcpyDeviceToHost));
    API_END
}

// Operator-level entry for the parity tests: one load-time weight kernel on caller buffers, launched as the build launches it.
int32_t b200rwkv_op_weight(int32_t device, int32_t kind, const b200rwkv_weight_args* args) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(args, B200RWKV_ERR_INVALID, "null arguments");
    REQUIRE(kind >= B200RWKV_WEIGHT_LORA && kind <= B200RWKV_WEIGHT_REPACK, B200RWKV_ERR_INVALID,
            "kind must be 0 (LoRA blend), 1 (f32 vector), 2 (decay table) or 3 (repack)");
    const b200rwkv_weight_args& x = *args;
    if (kind == B200RWKV_WEIGHT_LORA) {
        REQUIRE(x.w && x.lora_b && x.lora_a, B200RWKV_ERR_INVALID, "the LoRA blend needs w, lora_b and lora_a");
        REQUIRE(x.out >= 1 && x.in >= 1 && (int64_t)x.out * x.in <= ((int64_t)1 << 31) && x.r >= 1 && x.r <= 4096, B200RWKV_ERR_INVALID,
                "bad out / in / r (r must be 1..4096)");
    } else if (kind == B200RWKV_WEIGHT_REPACK) {
        REQUIRE(x.src && x.blocks, B200RWKV_ERR_INVALID, "the repack needs src and blocks");
        REQUIRE(x.rows >= 1 && x.ld >= 1 && (int64_t)x.rows * x.ld <= ((int64_t)1 << 31) && x.N >= 1 && x.K >= 1 && x.n0 >= 0 &&
                    x.k0 >= 0 && (int64_t)x.n0 + x.N <= x.rows && (int64_t)x.k0 + x.K <= x.ld,
                B200RWKV_ERR_INVALID, "the sub-matrix [n0, n0 + N) x [k0, k0 + K) must lie inside src [rows][ld]");
    } else {
        REQUIRE(x.src && x.dst && x.n >= 1 && x.n <= ((int64_t)1 << 30), B200RWKV_ERR_INVALID, "needs src, dst and n in 1..2^30");
    }
    CK(cudaSetDevice(device));
    int nsm = 0;
    CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    if (kind == B200RWKV_WEIGHT_LORA) {
        const size_t wb = (size_t)x.out * x.in * 2;
        Buf<__half> w(wb), b((size_t)x.out * x.r * 2), a((size_t)x.in * x.r * 2);
        CK(cudaMemcpy(w, x.w, wb, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(b, x.lora_b, (size_t)x.out * x.r * 2, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(a, x.lora_a, (size_t)x.in * x.r * 2, cudaMemcpyHostToDevice));
        launch_lora_blend(nsm, w, b, a, x.out, x.in, x.r, x.alpha);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(x.w, w, wb, cudaMemcpyDeviceToHost));
    } else if (kind == B200RWKV_WEIGHT_REPACK) {
        const size_t sb = (size_t)x.rows * x.ld * 2;
        const size_t db = (size_t)cdiv(x.N, GEMM_BN) * cdiv(x.K, GEMM_BK) * GEMM_WBYTES;
        Buf<__half> s(sb);
        Buf<uint8_t> d(db);
        CK(cudaMemcpy(s, x.src, sb, cudaMemcpyHostToDevice));
        CK(cudaMemset(d, 0xFF, db));               // a chunk the kernel leaves unwritten shows as NaN bits
        launch_repack(nsm, s, x.ld, x.n0, x.k0, x.N, x.K, reinterpret_cast<uint4*>(d.p));
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(x.blocks, d, db, cudaMemcpyDeviceToHost));
    } else {
        const size_t n = (size_t)x.n;
        Buf<__half> s(n * 2);
        Buf<float> d(n * 4);
        CK(cudaMemcpy(s, x.src, n * 2, cudaMemcpyHostToDevice));
        if (kind == B200RWKV_WEIGHT_F32) launch_f16_to_f32(s, d, n, x.scale, x.bias);
        else launch_decay_table(s, d, (int)n);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(x.dst, d, n * 4, cudaMemcpyDeviceToHost));
    }
    API_END
}

int32_t b200rwkv_launch_count(b200rwkv_engine* e, int64_t* total) {
    API_BEGIN(e)
    REQUIRE(e && total, B200RWKV_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    *total = (int64_t)e->launch_total;
    API_END
}

int32_t b200rwkv_keep_hidden(b200rwkv_engine* e, int32_t enable) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    e->hidden_keep = enable != 0;
    e->hidden_rows = 0;
    API_END
}

// returns the number of rows written (negative status on error)
int32_t b200rwkv_last_hidden(b200rwkv_engine* e, float* out, size_t cap) {
    return api_count([&]() -> int32_t {
        REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(e->mu);
        CK(cudaSetDevice(e->dev));
        CK(cudaStreamSynchronize(e->stream));
        const bool all = e->hidden_keep && e->d_hidden_all;
        const int32_t rows = all ? e->hidden_rows : e->last_T;
        const size_t n = (size_t)rows * e->C;
        REQUIRE(n <= cap, B200RWKV_ERR_INVALID, "hidden buffer too small");
        if (n) CK(cudaMemcpy(out, all ? e->d_hidden_all : e->d_hidden, n * 4, cudaMemcpyDeviceToHost));
        return rows;
    });
}

int32_t b200rwkv_keep_hidden_layers(b200rwkv_engine* e, int32_t n, const int32_t* layers) {
    API_BEGIN(e)
    REQUIRE(n >= 0 && n <= b200rwkv_engine::HID_MAX_LAYERS, B200RWKV_ERR_INVALID,
            "keep_hidden_layers: n must be in [0, " + std::to_string(b200rwkv_engine::HID_MAX_LAYERS) + "]");
    REQUIRE(n == 0 || layers, B200RWKV_ERR_INVALID, "keep_hidden_layers: null layers");
    for (int i = 0; i < n; ++i) {
        REQUIRE(layers[i] >= 0, B200RWKV_ERR_INVALID, "keep_hidden_layers: negative layer " + std::to_string(layers[i]));
        REQUIRE(std::find(layers, layers + i, layers[i]) == layers + i, B200RWKV_ERR_INVALID,
                "keep_hidden_layers: layer " + std::to_string(layers[i]) + " is listed twice");
    }
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    for (int i = 0; i < n; ++i)
        REQUIRE(layers[i] < e->L, B200RWKV_ERR_INVALID,
                "keep_hidden_layers: layer " + std::to_string(layers[i]) + " is outside [0, " + std::to_string(e->L) + ")");
    CK(cudaSetDevice(e->dev));
    if (n > 0 && !e->hid_step) e->hid_step = (float*)e->dalloc((size_t)b200rwkv_engine::HID_MAX_LAYERS * e->maxT * e->C * 4);
    e->hid_layers.assign(layers, layers + n);
    e->upload_hid_tab();
    API_END
}

int32_t b200rwkv_keep_hidden_pooled(b200rwkv_engine* e, int32_t n, const int32_t* layers, int32_t mode) {
    API_BEGIN(e)
    REQUIRE(n >= 0 && n <= POOL_MAX_LAYERS, B200RWKV_ERR_INVALID,
            "keep_hidden_pooled: n must be in [0, " + std::to_string(POOL_MAX_LAYERS) + "]");
    REQUIRE(n == 0 || layers, B200RWKV_ERR_INVALID, "keep_hidden_pooled: null layers");
    REQUIRE(mode == B200RWKV_POOL_LAST || mode == B200RWKV_POOL_MEAN, B200RWKV_ERR_INVALID,
            "keep_hidden_pooled: unknown mode " + std::to_string(mode));
    for (int i = 0; i < n; ++i) {
        REQUIRE(layers[i] >= 0, B200RWKV_ERR_INVALID, "keep_hidden_pooled: negative layer " + std::to_string(layers[i]));
        REQUIRE(std::find(layers, layers + i, layers[i]) == layers + i, B200RWKV_ERR_INVALID,
                "keep_hidden_pooled: layer " + std::to_string(layers[i]) + " is listed twice");
    }
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    for (int i = 0; i < n; ++i)
        REQUIRE(layers[i] < e->L, B200RWKV_ERR_INVALID,
                "keep_hidden_pooled: layer " + std::to_string(layers[i]) + " is outside [0, " + std::to_string(e->L) + ")");
    CK(cudaSetDevice(e->dev));
    if (n > 0 && !e->pool_step) e->pool_step = (float*)e->dalloc((size_t)POOL_MAX_LAYERS * e->maxT * e->C * 4);
    if (n > 0 && !e->pool_rows) e->pool_rows = (float*)e->dalloc((size_t)POOL_MAX_LAYERS * e->S * e->C * 4);
    e->pool_layers.assign(layers, layers + n);
    e->pool_mode = mode;
    e->upload_hid_tab();
    API_END
}

int32_t b200rwkv_score_top(b200rwkv_engine* e, int32_t top_n) {
    API_BEGIN(e)
    REQUIRE(top_n >= 0 && top_n <= TOPK_MAX, B200RWKV_ERR_INVALID,
            "score_top: top_n must be in [0, " + std::to_string(TOPK_MAX) + "]");
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    std::lock_guard<std::mutex> lk(e->mu);
    REQUIRE(top_n == 0 || e->world == 1, B200RWKV_ERR_UNSUPPORTED, "score_top: not supported under tensor parallelism");
    REQUIRE(top_n == 0 || e->V <= TOPK_MAX_SEGS * TOPK_SEG, B200RWKV_ERR_UNSUPPORTED,
            "score_top: num_vocab > " + std::to_string(TOPK_MAX_SEGS * TOPK_SEG) + " is not supported");
    CK(cudaSetDevice(e->dev));
    if (top_n > 0 && !e->top_cand_x) {
        const size_t n = (size_t)std::max(e->S, e->maxT) * cdiv(e->V, TOPK_SEG) * TOPK_MAX;
        e->top_cand_x = (float*)e->dalloc(n * 4);
        e->top_cand_id = (unsigned*)e->dalloc(n * 4);
    }
    e->top_n = top_n;
    API_END
}

// The head's weight format from the next infer call on (the infer task's call, like update_weights); every refusal is
// decided on the host first
int32_t b200rwkv_head_format(b200rwkv_engine* e, int32_t quant_type) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(quant_type >= QT_NONE && quant_type <= QT_INT4, B200RWKV_ERR_INVALID,
            "head_format: unknown quant_type " + std::to_string(quant_type));
    REQUIRE(quant_type != 3 && quant_type != 5, B200RWKV_ERR_UNSUPPORTED,
            "head_format: quant_type must be NONE, Int8, NF4, FP8 or Int4 (SF4 is not implemented)");
    std::lock_guard<std::mutex> lk(e->mu);
    if (quant_type == e->qhead.plan.qtype) return B200RWKV_OK;
    if (quant_type != QT_NONE) {
        REQUIRE(e->world == 1 && !e->group, B200RWKV_ERR_UNSUPPORTED, "head_format: a quantised head runs on one GPU (no tensor parallelism)");
        REQUIRE(e->precision == 0, B200RWKV_ERR_UNSUPPORTED, "head_format: a quantised head runs with precision 0 (f16 operands)");
        REQUIRE(e->C % GEMM_BK == 0, B200RWKV_ERR_UNSUPPORTED, "head_format: a quantised head needs num_emb to be a multiple of 128");
        REQUIRE(e->n_adapters == 0 || e->s_head.nproj == 0, B200RWKV_ERR_UNSUPPORTED,
                "head_format: this engine's adapters plan the head (a head pair or a B200RWKV_TARGET_HEAD place)");
    }
    e->set_head_format(quant_type);
    API_END
}

// returns the number of scored tokens of the most recent infer call (negative status on error)
int32_t b200rwkv_last_score_top(b200rwkv_engine* e, uint32_t* ids_out, float* logprobs_out, size_t cap) {
    return api_count([&]() -> int32_t {
        REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
        std::lock_guard<std::mutex> lk(e->mu);
        REQUIRE(e->top_last_n > 0, B200RWKV_ERR_STATE, "last_score_top: the most recent infer call ran without score_top");
        const size_t rows = e->top_last_rows, n = rows * e->top_last_n;
        if (!ids_out && !logprobs_out) return (int32_t)rows;       // the row count only
        REQUIRE(ids_out && logprobs_out, B200RWKV_ERR_INVALID, "last_score_top: one output is NULL");
        REQUIRE(n <= cap, B200RWKV_ERR_INVALID, "last_score_top: buffer too small");
        const uint8_t* h = e->sc_host + rows * (sizeof(ScoreRow) + 8);
        memcpy(ids_out, h, n * 4);
        memcpy(logprobs_out, h + n * 4, n * 4);
        return (int32_t)rows;
    });
}

// returns the number of rows written, one per entry of the call (negative status on error)
int32_t b200rwkv_last_hidden_pooled(b200rwkv_engine* e, int32_t layer, float* out, size_t cap, int32_t* ntok_out) {
    return api_count([&]() -> int32_t {
        REQUIRE(layer >= 0, B200RWKV_ERR_INVALID, "last_hidden_pooled: negative layer " + std::to_string(layer));
        REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(e->mu);
        REQUIRE(layer < e->L, B200RWKV_ERR_INVALID,
                "last_hidden_pooled: layer " + std::to_string(layer) + " is outside [0, " + std::to_string(e->L) + ")");
        const auto it = std::find(e->pool_last.begin(), e->pool_last.end(), layer);
        REQUIRE(it != e->pool_last.end(), B200RWKV_ERR_STATE,
                "last_hidden_pooled: layer " + std::to_string(layer) + " was not pooled by the most recent infer call");
        const size_t rows = e->pool_last_ntok.size(), C = (size_t)e->C;
        REQUIRE(rows * C <= cap, B200RWKV_ERR_INVALID, "last_hidden_pooled: buffer too small");
        CK(cudaSetDevice(e->dev));
        CK(cudaStreamSynchronize(e->stream));
        if (rows)
            CK(cudaMemcpy(out, e->pool_rows + (size_t)(it - e->pool_last.begin()) * e->S * C, rows * C * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < rows; ++i) {
            if (e->pool_last_ntok[i] == 0) std::fill_n(out + i * C, C, 0.f);      // no step held the entry: its row was not written
            if (ntok_out) ntok_out[i] = e->pool_last_ntok[i];
        }
        return (int32_t)rows;
    });
}

// returns the number of rows written (negative status on error)
int32_t b200rwkv_last_hidden_layer(b200rwkv_engine* e, int32_t layer, float* out, size_t cap) {
    return api_count([&]() -> int32_t {
        REQUIRE(layer >= 0, B200RWKV_ERR_INVALID, "last_hidden_layer: negative layer " + std::to_string(layer));
        REQUIRE(e && out, B200RWKV_ERR_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(e->mu);
        REQUIRE(layer < e->L, B200RWKV_ERR_INVALID,
                "last_hidden_layer: layer " + std::to_string(layer) + " is outside [0, " + std::to_string(e->L) + ")");
        const auto it = std::find(e->hid_last.begin(), e->hid_last.end(), layer);
        REQUIRE(it != e->hid_last.end(), B200RWKV_ERR_STATE,
                "last_hidden_layer: layer " + std::to_string(layer) + " was not recorded by the most recent infer call");
        const size_t n = e->hid_last_rows * e->C;
        REQUIRE(n <= cap, B200RWKV_ERR_INVALID, "last_hidden_layer: buffer too small");
        CK(cudaSetDevice(e->dev));
        CK(cudaStreamSynchronize(e->stream));
        if (n) CK(cudaMemcpy(out, e->hid_all + (size_t)(it - e->hid_last.begin()) * n, n * 4, cudaMemcpyDeviceToHost));
        return (int32_t)e->hid_last_rows;
    });
}

// Debug aid for the parity tests: copy a named internal activation buffer of the most recent
// step to the host as f32 row-major [rows, cols]; returns cols (rows = tokens of the last step,
// capped by `cap`), or a negative status.  Not used on the product path.
int32_t b200rwkv_debug_read(b200rwkv_engine* e, const char* name, float* out, size_t cap) {
    return api_count([&]() -> int32_t {
        REQUIRE(e && name && out, B200RWKV_ERR_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(e->mu);
        CK(cudaSetDevice(e->dev));
        CK(cudaStreamSynchronize(e->stream));
        const std::string n(name);
        const int T = std::max(e->last_T, 1);
        struct F { const char* n; float* p; int cols; };
        const F fs[] = {{"x_a", e->x_a, e->C}, {"x_b", e->x_b, e->C}, {"xx1", e->xx1, e->C}, {"sx1", e->sx1, e->C}, {"xx2", e->xx2, e->C},
                        {"r", e->f_r, e->Cl}, {"k", e->f_k, e->Cl}, {"v", e->f_v, e->Cl}, {"g", e->f_g, e->Cl}, {"w", e->f_w, e->Cl},
                        {"a", e->f_a, e->Cl}, {"nu", e->f_nu, e->Cl}, {"v_first", e->f_vfirst, e->Cl}, {"rr", e->f_rr, e->Cl},
                        {"part_att", e->part_att, e->C},
                        {"part_ffn", e->part_ffn, e->C}, {"hidden", e->d_hidden, e->C}};
        for (const F& f : fs)
            if (n == f.n) {
                REQUIRE((size_t)T * f.cols <= cap, B200RWKV_ERR_INVALID, "debug buffer too small");
                CK(cudaMemcpy(out, f.p, (size_t)T * f.cols * 4, cudaMemcpyDeviceToHost));
                const int nsum = (n == "part_att") ? e->split_att : (n == "part_ffn" ? e->split_ffn : 1);
                std::vector<float> tmp((size_t)T * f.cols);
                for (int sp = 1; sp < nsum; ++sp) {       // split-K partials: sum the slices
                    CK(cudaMemcpy(tmp.data(), f.p + (size_t)sp * e->maxT * e->C, tmp.size() * 4, cudaMemcpyDeviceToHost));
                    for (size_t i = 0; i < tmp.size(); ++i) out[i] += tmp[i];
                }
                return f.cols;
            }
        if (n.rfind("hid_step", 0) == 0 && n.size() == 9 && n[8] >= '0' && n[8] < '0' + b200rwkv_engine::HID_MAX_LAYERS) {
            // step buffer k of b200rwkv_keep_hidden_layers (zeros until the first layer is recorded into it)
            REQUIRE(e->hid_step, B200RWKV_ERR_STATE, "no hidden layer has been recorded yet");
            REQUIRE((size_t)T * e->C <= cap, B200RWKV_ERR_INVALID, "debug buffer too small");
            CK(cudaMemcpy(out, e->hid_step + (size_t)(n[8] - '0') * e->maxT * e->C, (size_t)T * e->C * 4, cudaMemcpyDeviceToHost));
            return e->C;
        }
        struct A { std::string n; const A16Buf* b; int cols; int mat; };
        std::vector<A> as;
        for (int i = 0; i < 6; ++i) as.push_back({"a_x" + std::to_string(i), &e->a_x[i], e->C, 0});
        for (int i = 0; i < 5; ++i)
            for (int m = 0; m < 5; ++m)
                as.push_back({"a_lora" + std::to_string(i) + "_" + std::to_string(m), &e->a_lora[i],
                              (int)(e->a_lora[i].halves_per_matrix / A16_KB_HALVES) * GEMM_BK, m});
        as.push_back({"a_out", &e->a_out, e->Cl, 0});
        as.push_back({"a_kk", &e->a_kk, e->Fl, 0});
        as.push_back({"a_head", &e->a_head, e->C, 0});
        // "<buffer>_lo": the lo halves of a split operand (token rows 16..31), after a step that ran split operands;
        // "<buffer>_tail" (and "_tail_lo"): the n_adapters 128-wide adapter tail blocks of a projection operand, which start
        // at its own columns rounded up to whole k blocks
        auto strip = [](std::string& s, const char* suf) {
            const size_t k = strlen(suf);
            const bool has = s.size() > k && s.compare(s.size() - k, k, suf) == 0;
            if (has) s.resize(s.size() - k);
            return has;
        };
        std::string base = n;
        const bool lo = strip(base, "_lo");
        const bool tail = strip(base, "_tail");
        for (const A& a : as)
            if (base == a.n && a.b->p) {
                REQUIRE(!tail || (e->n_adapters && base.rfind("a_lora", 0) != 0), B200RWKV_ERR_STATE,
                        "debug_read: " + base + " has no adapter tail blocks (an engine with adapters, a projection operand)");
                REQUIRE(!lo || e->last_sh.split, B200RWKV_ERR_STATE, "debug_read: the last step did not run split operands, " + n + " has no lo half");
                const int k0 = tail ? cdiv(a.cols, GEMM_BK) * GEMM_BK : 0, cols = tail ? e->n_adapters * GEMM_BK : a.cols;
                REQUIRE((size_t)T * cols <= cap, B200RWKV_ERR_INVALID, "debug buffer too small");
                // the head's operand holds the step's output rows (th_rows), every other operand its token rows (th)
                const int tr = (a.b == &e->a_head) ? e->last_sh.th_rows : e->last_sh.th, r0 = lo ? 16 : 0;
                std::vector<uint16_t> h(a.b->halves_per_matrix);
                CK(cudaMemcpy(h.data(), a.b->p + (size_t)a.mat * a.b->halves_per_matrix, h.size() * 2, cudaMemcpyDeviceToHost));
                // a16_index does not depend on the operand's width: column k0 + k is the unpack's column k shifted
                for (int m = 0; m < T; ++m)
                    for (int k = 0; k < cols; ++k)
                        out[(size_t)m * cols + k] = __half2float(__ushort_as_half(h[a16_index(r0 + m, k0 + k, tr)]));
                return cols;
            }
        throw Error(B200RWKV_ERR_INVALID, "unknown debug buffer: " + n);
    });
}

// Test aid: the weight fills of one tensor (b200rwkv_debug_fills), and one of them read back (b200rwkv_debug_fill).  Not used
// on the product path.
int32_t b200rwkv_debug_fills(b200rwkv_engine* e, const char* name) {
    return api_count([&]() -> int32_t {
        REQUIRE(e && name, B200RWKV_ERR_INVALID, "null argument");
        std::lock_guard<std::mutex> lk(e->mu);
        const auto it = e->fills.find(name);
        return it == e->fills.end() ? 0 : (int32_t)it->second.size();
    });
}

int32_t b200rwkv_debug_fill(b200rwkv_engine* e, const char* name, int32_t i, b200rwkv_fill_info* info, void* out, size_t cap) {
    API_BEGIN(e)
    REQUIRE(e && name && info, B200RWKV_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(e->mu);
    const auto it = e->fills.find(name);
    REQUIRE(it != e->fills.end(), B200RWKV_ERR_INVALID, std::string("debug_fill: the engine fills nothing from ") + name);
    REQUIRE(i >= 0 && i < (int32_t)it->second.size(), B200RWKV_ERR_INVALID,
            "debug_fill: " + std::string(name) + " has " + std::to_string(it->second.size()) + " fills, no fill " + std::to_string(i));
    const Fill& f = it->second[i];
    const size_t R = (size_t)f.tiles * GEMM_BN, Kp = (size_t)f.kb * GEMM_BK;
    size_t bytes = 0, param_bytes = 0;
    switch (f.kind) {
        case FILL_SEG:
            param_bytes = f.qtype == QT_FP8 ? R * 4 : f.qtype == QT_INT8 || f.qtype == QT_INT4 || f.qtype == QT_NF4 ? R * f.kb * 4 : 0;
            bytes = R * Kp * (f.qtype == QT_NONE ? 2 : 1) + param_bytes + R * f.ad_tail * GEMM_BK * 2;
            break;
        case FILL_VEC: case FILL_DECAY: bytes = f.count * 4; break;
        case FILL_RAW: bytes = f.count * 2; break;
        case FILL_FOLD: bytes = (size_t)f.N * f.K * 64 * 2; break;
        default: bytes = (size_t)(e->N + 2) * e->C * 4; break;          // FILL_INIT
    }
    REQUIRE(!out || cap >= bytes, B200RWKV_ERR_INVALID, "debug_fill: the buffer holds " + std::to_string(cap) + " bytes, the fill " +
            std::to_string(bytes));
    b200rwkv_fill_info fi;
    memset(&fi, 0, sizeof(fi));
    fi.kind = f.kind; fi.qtype = f.qtype; fi.plan = f.plan;
    fi.n0 = f.kind == FILL_INIT ? f.layer : f.n0; fi.N = f.N; fi.k0 = f.k0; fi.K = f.K; fi.ld = f.ld; fi.off = (int64_t)f.off;
    fi.tiles = f.tiles; fi.kb = f.kb; fi.ad_tail = f.ad_tail; fi.count = (int64_t)f.count; fi.scale = f.scale; fi.bias = f.bias;
    fi.bytes = bytes;
    *info = fi;
    if (!out) return B200RWKV_OK;
    uint8_t* o = static_cast<uint8_t*>(out);
    if (f.kind == FILL_INIT) {
        REQUIRE(!e->init_state.empty(), B200RWKV_ERR_INVALID, "internal: a time_state fill without State::init rows");
        memcpy(o, e->init_state.data() + (size_t)f.layer * (e->N + 2) * e->C, bytes);
        return B200RWKV_OK;
    }
    CK(cudaSetDevice(e->dev));
    CK(cudaStreamSynchronize(e->stream));
    if (f.kind != FILL_SEG) {
        CK(cudaMemcpy(o, f.dst, bytes, cudaMemcpyDeviceToHost));
        return B200RWKV_OK;
    }
    if (f.qtype == QT_NONE) {
        std::vector<uint16_t> h((size_t)f.tiles * f.dst_kb * GEMM_WBYTES / 2);
        CK(cudaMemcpy(h.data(), f.dst, h.size() * 2, cudaMemcpyDeviceToHost));
        untile_f16(h.data(), f.tiles, f.dst_kb, 0, f.kb, reinterpret_cast<uint16_t*>(o));
        o += R * Kp * 2;
    } else {
        std::vector<uint8_t> h((size_t)f.tiles * f.kb * q_block_bytes(f.qtype));
        CK(cudaMemcpy(h.data(), f.dst, h.size(), cudaMemcpyDeviceToHost));
        uint16_t* p0 = reinterpret_cast<uint16_t*>(o + R * Kp);
        if (f.qtype == QT_FP8) CK(cudaMemcpy(p0, f.scales, R * 4, cudaMemcpyDeviceToHost));
        untile_codes(f.qtype, h.data(), f.tiles, f.kb, (int)R, o, p0, p0 + R * f.kb);
        o += R * Kp + param_bytes;
    }
    if (f.ad_tail) {
        std::vector<uint16_t> h((size_t)f.tiles * f.ad_tail * GEMM_WBYTES / 2);
        CK(cudaMemcpy2D(h.data(), (size_t)f.ad_tail * GEMM_WBYTES, f.tails, (size_t)f.tails_kb * GEMM_WBYTES,
                        (size_t)f.ad_tail * GEMM_WBYTES, f.tiles, cudaMemcpyDeviceToHost));
        untile_f16(h.data(), f.tiles, f.ad_tail, 0, f.ad_tail, reinterpret_cast<uint16_t*>(o));
    }
    API_END
}

// Profiling aid: the raw stamp rows of the most recent traced replay (b200rwkv_profile_insitu): one row of 512 uint64 per
// launch -- [0..7] globaltimer stamps of CTA 0 (entry, past griddepcontrol.wait, phase marks, exit), then {SM id, last MMA
// issued, exit} of every projection CTA (or {entry, released, phase 1 done} of every CTA of the RWKV-6 front-half kernel).
int32_t b200rwkv_debug_trace(b200rwkv_engine* e, uint64_t* out, size_t cap, int32_t* types, int32_t* nphase) {
    API_BEGIN(e)
    REQUIRE(e && out && types && nphase, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(e->d_step_trace && !e->step_trace_types.empty(), B200RWKV_ERR_INVALID, "no trace: call b200rwkv_profile_insitu first");
    std::lock_guard<std::mutex> lk(e->mu);
    const size_t nl = e->step_trace_types.size();
    const size_t row = b200rwkv_engine::STEP_TRACE_ROW;
    REQUIRE(cap >= nl * row, B200RWKV_ERR_INVALID, "trace buffer too small");
    CK(cudaSetDevice(e->dev));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(out, e->d_step_trace, nl * row * 8, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < nl; ++i) types[i] = e->step_trace_types[i];
    *nphase = (int32_t)nl;
    API_END
}

// Profiling aid: time one projection launch class in isolation, round-robin over the layers so
// every launch streams cold weights.  which: 0.. = the launches between LN1 and WKV of a step of
// more than 16 tokens (the ddlerp LoRA launches first), 10 = output projection, 20.. = channel-mix
// launches, 30 = head; any other index is refused.  Returns ms per launch and weight bytes.
int32_t b200rwkv_debug_gemm_time(b200rwkv_engine* e, int32_t which, int32_t reps, float* ms_out, int64_t* bytes_out,
                                 uint64_t* trace_out /* [L][8] stamps of CTA 0 for the last round, or null */) {
    API_BEGIN(e)
    REQUIRE(e && ms_out && bytes_out && reps >= 1, B200RWKV_ERR_INVALID, "bad argument");
    std::lock_guard<std::mutex> lk(e->mu);
    CK(cudaSetDevice(e->dev));
    auto pick = [&](int l) -> const GemmLaunch& {
        const Layer& ly = e->layers[l % e->L];
        const int nl = (int)ly.lora.size(), np = (int)ly.pre.size(), nf = (int)ly.ffn.size();
        if (which == 30) return e->head_plan(false);
        if (which == 10) return ly.o;
        if (which >= 20 && which < 20 + nf) return ly.ffn[which - 20];
        REQUIRE(which >= 0 && which < nl + np, B200RWKV_ERR_INVALID, "no such launch");
        return which < nl ? ly.lora[which] : ly.pre[which - nl];
    };
    // a valid 16-token meta so row masks are full
    std::vector<int> m(e->meta_ints, 0);
    m[0] = 16; m[1] = std::min(16, e->S); m[2] = 16;
    CK(cudaMemcpy(e->d_meta, m.data(), e->meta_ints * 4, cudaMemcpyHostToDevice));
    Event a = new_event(), b = new_event();
    const int n = reps * e->L;
    Buf<unsigned long long> d_tr;
    if (trace_out) { d_tr = Buf<unsigned long long>((size_t)e->L * 16 * 8); CK(cudaMemset(d_tr, 0, (size_t)e->L * 16 * 8)); }
    const StepShape sh = e->step_shape(16, 16);
    for (int i = 0; i < e->L; ++i) e->launch_gemm(pick(i), sh, e->stream, nullptr);
    CK(cudaEventRecord(a, e->stream));
    for (int i = 0; i < n; ++i) {
        GemmLaunch g = pick(i);
        if (d_tr && i >= n - e->L) g.p.trace = d_tr + (size_t)(i % e->L) * 16;
        e->launch_gemm(g, sh, e->stream, nullptr);
    }
    CK(cudaEventRecord(b, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (d_tr) CK(cudaMemcpy(trace_out, d_tr, (size_t)e->L * 16 * 8, cudaMemcpyDeviceToHost));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, a, b));
    *ms_out = ms / n;
    *bytes_out = (int64_t)pick(0).weight_bytes;
    API_END
}

// ---- exported SPMD entries: one rank, or all ranks of an in-process tensor-parallel engine at once ----
#define RANKS(e, call_r) ((e) && (e)->group ? (e)->group->spmd([&](int r_) -> int32_t { b200rwkv_engine* er = (e)->group->ranks[r_]; (void)er; return call_r; }) : [&]() -> int32_t { b200rwkv_engine* er = (e); const int r_ = 0; (void)r_; return call_r; }())

int32_t b200rwkv_infer(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const int32_t* ntok, const uint32_t* tokens,
                       const int32_t* option, float* logits_out, size_t logits_cap, int32_t* rows_out) {
    return RANKS(e, rank_infer(er, nslot, slot, ntok, tokens, option, r_ == 0 ? logits_out : nullptr, r_ == 0 ? logits_cap : 0,
                               r_ == 0 ? rows_out : nullptr));
}
static int32_t check_infer_args(const b200rwkv_infer_args* a) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(a, B200RWKV_ERR_INVALID, "infer_ex: null args");
    REQUIRE(a->struct_bytes == sizeof(b200rwkv_infer_args), B200RWKV_ERR_INVALID,
            "infer_ex: struct_bytes is " + std::to_string(a->struct_bytes) + ", expected sizeof(b200rwkv_infer_args) = " +
            std::to_string(sizeof(b200rwkv_infer_args)));
    API_END
}
int32_t b200rwkv_infer_ex(b200rwkv_engine* e, const b200rwkv_infer_args* a) {
    const int32_t st = check_infer_args(a);
    if (st < 0) return st;
    const b200rwkv_engine::ScoreOut sc{a->score_out, a->argmax_out};
    return RANKS(e, rank_infer(er, a->nslot, a->slot, a->ntok, a->tokens, a->option, r_ == 0 ? a->logits_out : nullptr,
                               r_ == 0 ? a->logits_cap : 0, r_ == 0 ? a->rows_out : nullptr, &sc));
}
int32_t b200rwkv_infer_snapshots(b200rwkv_engine* e, const b200rwkv_infer_args* a, int32_t nsnap, const int32_t* snap_entry,
                                 const int32_t* snap_tokens, uint64_t* snap_ids) {
    const int32_t st = check_infer_args(a);
    if (st < 0) return st;
    // both tensor-parallel front ends go through every rank's b200rwkv_engine::infer, which refuses snapshots (nsnap > 0) on a
    // rank of a world above 1 after infer_ex's own checks; nsnap == 0 runs as infer_ex
    const b200rwkv_engine::ScoreOut sc{a->score_out, a->argmax_out};
    const b200rwkv_engine::SnapPlan sp{nsnap, snap_entry, snap_tokens, snap_ids};
    return RANKS(e, rank_infer(er, a->nslot, a->slot, a->ntok, a->tokens, a->option, r_ == 0 ? a->logits_out : nullptr,
                               r_ == 0 ? a->logits_cap : 0, r_ == 0 ? a->rows_out : nullptr, &sc, &sp));
}
int32_t b200rwkv_state_load(b200rwkv_engine* e, int32_t slot, const float* in) { return RANKS(e, rank_state_load(er, slot, in)); }

// head-sharded state: every rank exports the WKV rows of its own heads (zeros elsewhere); the shift rows are replicated
static void merge_state_columns(const b200rwkv_engine* lead, float* out, const float* part, int r) {
    const int C = lead->C, N = lead->N, Cl = lead->Cl;
    for (int l = 0; l < lead->L; ++l)
        for (int row = 1; row <= N; ++row) {
            const size_t o = ((size_t)l * (N + 2) + row) * C + (size_t)r * Cl;
            memcpy(out + o, part + o, (size_t)Cl * 4);
        }
}
int32_t b200rwkv_state_back(b200rwkv_engine* e, int32_t slot, float* out) {
    if (!e || !e->group) return rank_state_back(e, slot, out);
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    std::vector<std::vector<float>> part(e->group->ranks.size());
    for (size_t r = 1; r < part.size(); ++r) part[r].resize(n);
    const int32_t st = e->group->spmd([&](int r) { return rank_state_back(e->group->ranks[r], slot, r == 0 ? out : part[r].data()); });
    if (st < 0 || !out) return st;
    for (size_t r = 1; r < part.size(); ++r) merge_state_columns(e, out, part[r].data(), (int)r);
    return st;
}
int32_t b200rwkv_state_read(b200rwkv_engine* e, int32_t slot, uint64_t* snapshot_id) {
    if (!e || !e->group) return rank_state_read(e, slot, snapshot_id);
    // every rank snapshots its shard; the ranks' id counters advance in lockstep, so the ids agree
    std::vector<uint64_t> ids(e->group->ranks.size(), 0);
    const int32_t st = e->group->spmd([&](int r) { return rank_state_read(e->group->ranks[r], slot, &ids[r]); });
    if (st < 0) return st;
    for (uint64_t id : ids)
        if (id != ids[0]) { g_err = "internal: snapshot ids diverged across ranks"; return B200RWKV_ERR_STATE; }
    if (snapshot_id) *snapshot_id = ids[0];
    return st;
}
int32_t b200rwkv_state_write(b200rwkv_engine* e, int32_t slot, uint64_t id) { return RANKS(e, rank_state_write(er, slot, id)); }
int32_t b200rwkv_state_free(b200rwkv_engine* e, uint64_t id) { return RANKS(e, rank_state_free(er, id)); }
int32_t b200rwkv_snapshot_back(b200rwkv_engine* e, uint64_t id, float* state_out, float* logits_out) {
    if (!e || !e->group) return rank_snapshot_back(e, id, state_out, logits_out);
    const size_t n = (size_t)e->L * (e->N + 2) * e->C;
    std::vector<std::vector<float>> part(e->group->ranks.size());
    for (size_t r = 1; r < part.size(); ++r) part[r].resize(state_out ? n : 0);
    const int32_t st = e->group->spmd([&](int r) {
        if (r == 0) return rank_snapshot_back(e, id, state_out, logits_out);
        return state_out ? rank_snapshot_back(e->group->ranks[r], id, part[r].data(), nullptr) : (int32_t)B200RWKV_OK;
    });
    if (st < 0 || !state_out) return st;
    for (size_t r = 1; r < part.size(); ++r) merge_state_columns(e, state_out, part[r].data(), (int)r);
    return st;
}
int32_t b200rwkv_snapshot_load(b200rwkv_engine* e, const float* state_in, const float* logits_in, uint64_t* snapshot_id) {
    if (!e || !e->group) return rank_snapshot_load(e, state_in, logits_in, snapshot_id);
    std::vector<uint64_t> ids(e->group->ranks.size(), 0);
    const int32_t st = e->group->spmd([&](int r) { return rank_snapshot_load(e->group->ranks[r], state_in, r == 0 ? logits_in : nullptr, &ids[r]); });
    if (st < 0) return st;
    for (uint64_t id : ids)
        if (id != ids[0]) { g_err = "internal: snapshot ids diverged across ranks"; return B200RWKV_ERR_STATE; }
    if (snapshot_id) *snapshot_id = ids[0];
    return st;
}
int32_t b200rwkv_bench_decode(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int32_t warmup,
                              int32_t steps, int32_t flush_l2, float* ms_out, int64_t* launches_out, float* step_ms_out) {
    if (!e || !e->group) return rank_bench_decode(e, nslot, slot, tokens, warmup, steps, flush_l2, ms_out, launches_out, step_ms_out);
    const size_t W = e->group->ranks.size();
    std::vector<float> ms(W, 0.f);
    std::vector<int64_t> ln(W, 0);
    const int32_t st = e->group->spmd([&](int r) {
        return rank_bench_decode(e->group->ranks[r], nslot, slot, tokens, warmup, steps, flush_l2, &ms[r], &ln[r], r == 0 ? step_ms_out : nullptr);
    });
    if (st < 0) return st;
    if (ms_out) *ms_out = *std::max_element(ms.begin(), ms.end());        // a step is done when the slowest rank is
    if (launches_out) *launches_out = ln[0];
    return st;
}
int32_t b200rwkv_profile_step(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, float ms[4],
                              int32_t launches[4], int64_t* gemm_weight_bytes) {
    if (!e || !e->group) return rank_profile_step(e, nslot, slot, tokens, ms, launches, gemm_weight_bytes);
    const size_t W = e->group->ranks.size();
    std::vector<float> m4(4 * W);
    std::vector<int32_t> l4(4 * W);
    std::vector<int64_t> wb(W);
    const int32_t st = e->group->spmd([&](int r) { return rank_profile_step(e->group->ranks[r], nslot, slot, tokens, &m4[4 * r], &l4[4 * r], &wb[r]); });
    if (st < 0) return st;
    for (int i = 0; i < 4; ++i) { ms[i] = m4[i]; launches[i] = l4[i]; }
    if (gemm_weight_bytes) *gemm_weight_bytes = wb[0];
    return st;
}
int32_t b200rwkv_profile_insitu(b200rwkv_engine* e, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int32_t reps,
                                int32_t cap, int32_t* n_out, int32_t* types, double* start_us, double* end_us, int64_t* bytes,
                                double* step_us) {
    if (!e || !e->group) return rank_profile_insitu(e, nslot, slot, tokens, reps, cap, n_out, types, start_us, end_us, bytes, step_us);
    const size_t W = e->group->ranks.size();
    std::vector<std::vector<int32_t>> ty(W, std::vector<int32_t>(cap));
    std::vector<std::vector<double>> su(W, std::vector<double>(cap)), eu(W, std::vector<double>(cap));
    std::vector<std::vector<int64_t>> by(W, std::vector<int64_t>(cap));
    std::vector<int32_t> nn(W, 0);
    std::vector<double> sus(W, 0.0);
    const int32_t st = e->group->spmd([&](int r) {
        if (r == 0) return rank_profile_insitu(e, nslot, slot, tokens, reps, cap, n_out, types, start_us, end_us, bytes, step_us);
        return rank_profile_insitu(e->group->ranks[r], nslot, slot, tokens, reps, cap, &nn[r], ty[r].data(), su[r].data(), eu[r].data(), by[r].data(), &sus[r]);
    });
    return st;
}
#undef RANKS

// Replaces `ModelBuilder...build_vN()` + `Bundle::new` + `TokioRuntime::new` (lib.rs:484-497) with everything the reference's
// ReloadRequest carries for this path: devices (one engine object owning all tensor-parallel ranks, SURVEY.md §8b), LoRA files
// (lib.rs:466-485), precision (lib.rs:493).
// b200rwkv_options as this library reads it: both sizes the header has had (the one before `batch_invariant` leaves both
// flags off; `quant_adapters` fills the tail padding of the current size), every value checked before any CUDA call
static int32_t read_options(const b200rwkv_options* opt, bool* batch_inv, bool* quant_adapters = nullptr) {
    if (opt->struct_bytes != sizeof(b200rwkv_options) && opt->struct_bytes != offsetof(b200rwkv_options, batch_invariant)) {
        g_err = "b200rwkv_options.struct_bytes does not match this library";
        return B200RWKV_ERR_INVALID;
    }
    const bool full = opt->struct_bytes == sizeof(b200rwkv_options);
    const int32_t bi = full ? opt->batch_invariant : 0;
    const int32_t qa = full ? opt->quant_adapters : 0;
    if (bi != 0 && bi != 1) { g_err = "b200rwkv_options.batch_invariant must be 0 or 1"; return B200RWKV_ERR_INVALID; }
    if (qa != 0 && qa != 1) { g_err = "b200rwkv_options.quant_adapters must be 0 or 1"; return B200RWKV_ERR_INVALID; }
    if (bi && opt->num_devices > 1) { g_err = "the batch-invariant mode runs on one GPU (no tensor parallelism)"; return B200RWKV_ERR_UNSUPPORTED; }
    if (qa && opt->num_devices > 1) { g_err = "adapters on quantised layers run on one GPU (no tensor parallelism)"; return B200RWKV_ERR_UNSUPPORTED; }
    *batch_inv = bi != 0;
    if (quant_adapters) *quant_adapters = qa != 0;
    return B200RWKV_OK;
}

int32_t b200rwkv_create_ex(const uint8_t* st, size_t len, const b200rwkv_options* opt, b200rwkv_engine** out) {
    if (!out || !opt) { g_err = "null argument"; return B200RWKV_ERR_INVALID; }
    *out = nullptr;
    bool batch_inv = false;
    if (const int32_t rc = read_options(opt, &batch_inv)) return rc;
    const int world = opt->num_devices <= 0 ? 1 : opt->num_devices;
    if (!(world == 1 || world == 2 || world == 4 || world == 8)) { g_err = "num_devices must be 1, 2, 4 or 8"; return B200RWKV_ERR_INVALID; }
    if (opt->num_lora < 0 || opt->num_lora > B200RWKV_MAX_LORA) { g_err = "bad num_lora"; return B200RWKV_ERR_INVALID; }
    std::vector<LoraArg> lora;
    for (int i = 0; i < opt->num_lora; ++i) lora.push_back({opt->lora_st[i], opt->lora_len[i], opt->lora_alpha[i]});
    const int dev0 = opt->num_devices <= 0 ? 0 : opt->devices[0];
    if (world == 1)
        return create_rank(st, len, dev0, opt->max_batch, opt->token_chunk_size, opt->precision, 0, 1, lora, out, opt->quant_layers, opt->quant_type,
                           {}, 0, 0, batch_inv);
    if (opt->quant_layers > 0 && opt->quant_type != B200RWKV_QUANT_NONE) { g_err = "quantised layers are single-GPU in this version"; return B200RWKV_ERR_UNSUPPORTED; }
    for (int r = 0; r < world; ++r)
        for (int q = 0; q < r; ++q)
            if (opt->devices[r] == opt->devices[q]) { g_err = "devices must be distinct"; return B200RWKV_ERR_INVALID; }
    // build all ranks concurrently (each uploads and re-tiles its own shard), then wire them
    std::unique_ptr<Group> g(new Group());
    g->ranks.assign(world, nullptr);
    g->start(world);
    const int32_t st_build = g->spmd([&](int r) {
        return create_rank(st, len, opt->devices[r], opt->max_batch, opt->token_chunk_size, opt->precision, r, world, lora, &g->ranks[r]);
    });
    int32_t rc = st_build;
    if (rc >= 0) rc = b200rwkv_tp_connect_local(g->ranks.data(), world);
    if (rc < 0) {
        const std::string msg = g_err;
        g->shutdown();
        for (auto* p : g->ranks) delete p;
        g_err = msg;
        return rc;
    }
    b200rwkv_engine* lead = g->ranks[0];
    lead->group = std::move(g);
    *out = lead;
    return B200RWKV_OK;
}

// b200rwkv_create_ex with unblended adapters: everything about the files is checked on the host before any CUDA call
int32_t b200rwkv_create_adapters(const uint8_t* st, size_t len, const b200rwkv_options* opt, int32_t n, const uint8_t* const* adapter_st,
                                 const size_t* adapter_len, const float* adapter_alpha, b200rwkv_engine** out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(out && opt, B200RWKV_ERR_INVALID, "null argument");
    *out = nullptr;
    bool quant_adapters = false;
    {
        bool batch_inv = false;
        if (const int32_t rc = read_options(opt, &batch_inv, &quant_adapters)) return rc;
        // a bound step runs W' plans with another K split: an unbound slot's bits would depend on its neighbours' bindings
        REQUIRE(!batch_inv, B200RWKV_ERR_UNSUPPORTED, "the batch-invariant mode does not run adapters");
    }
    const int refused_layers = quant_adapters ? 0 : opt->quant_layers;     // layers whose matrices adapters may not pair
    REQUIRE(n >= 1 && n <= AD_MAX, B200RWKV_ERR_INVALID, "number of adapters must be 1..8");
    REQUIRE(adapter_st && adapter_len && adapter_alpha, B200RWKV_ERR_INVALID, "null adapter list");
    REQUIRE(opt->num_devices <= 1, B200RWKV_ERR_UNSUPPORTED, "adapters run on one GPU (no tensor parallelism)");
    REQUIRE(opt->num_lora >= 0 && opt->num_lora <= B200RWKV_MAX_LORA, B200RWKV_ERR_INVALID, "bad num_lora");
    REQUIRE(opt->quant_layers >= 0 && opt->quant_type >= 0, B200RWKV_ERR_INVALID, "bad quant_layers / quant_type");
    StFile model(st, len);
    std::vector<std::unique_ptr<StFile>> files;
    std::vector<b200rwkv_engine::LoraSrc> srcs;
    for (int a = 0; a < n; ++a) {
        REQUIRE(adapter_st[a] && adapter_len[a] > 8, B200RWKV_ERR_INVALID, "null adapter image");
        files.emplace_back(new StFile(adapter_st[a], adapter_len[a]));
        srcs.push_back({files.back().get(), adapter_alpha[a]});
    }
    check_adapter_files(model.tensors, srcs, refused_layers, opt->quant_type);
    std::vector<LoraArg> lora;
    for (int i = 0; i < opt->num_lora; ++i) lora.push_back({opt->lora_st[i], opt->lora_len[i], opt->lora_alpha[i]});
    const int dev0 = opt->num_devices <= 0 ? 0 : opt->devices[0];
    return create_rank(st, len, dev0, opt->max_batch, opt->token_chunk_size, opt->precision, 0, 1, lora, out, opt->quant_layers,
                       opt->quant_type, srcs, 0, 0, false, quant_adapters);
    API_END
}

// b200rwkv_create_ex with n empty adapter places, W' plans for every targeted matrix of the f16 layers: checked on the host
// before any CUDA call
int32_t b200rwkv_create_adapter_places(const uint8_t* st, size_t len, const b200rwkv_options* opt, int32_t n, uint32_t targets,
                                       b200rwkv_engine** out) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(out && opt, B200RWKV_ERR_INVALID, "null argument");
    *out = nullptr;
    bool quant_adapters = false;
    {
        bool batch_inv = false;
        if (const int32_t rc = read_options(opt, &batch_inv, &quant_adapters)) return rc;
        // a bound step runs W' plans with another K split: an unbound slot's bits would depend on its neighbours' bindings
        REQUIRE(!batch_inv, B200RWKV_ERR_UNSUPPORTED, "the batch-invariant mode does not run adapters");
    }
    REQUIRE(n >= 1 && n <= AD_MAX, B200RWKV_ERR_INVALID, "number of adapter places must be 1..8");
    REQUIRE(targets != 0 && (targets & ~AD_TARGET_ALL) == 0, B200RWKV_ERR_INVALID,
            "adapter targets must be a nonzero set of B200RWKV_TARGET_* bits");
    REQUIRE(opt->num_devices <= 1, B200RWKV_ERR_UNSUPPORTED, "adapters run on one GPU (no tensor parallelism)");
    REQUIRE(opt->num_lora >= 0 && opt->num_lora <= B200RWKV_MAX_LORA, B200RWKV_ERR_INVALID, "bad num_lora");
    REQUIRE(opt->quant_layers >= 0 && opt->quant_type >= 0, B200RWKV_ERR_INVALID, "bad quant_layers / quant_type");
    StFile model(st, len);
    REQUIRE(!ad_place_matrices(model.tensors, targets, quant_adapters ? 0 : opt->quant_layers, opt->quant_type).empty(),
            B200RWKV_ERR_UNSUPPORTED, "adapter targets name no f16 projection matrix of this model");
    std::vector<LoraArg> lora;
    for (int i = 0; i < opt->num_lora; ++i) lora.push_back({opt->lora_st[i], opt->lora_len[i], opt->lora_alpha[i]});
    const int dev0 = opt->num_devices <= 0 ? 0 : opt->devices[0];
    return create_rank(st, len, dev0, opt->max_batch, opt->token_chunk_size, opt->precision, 0, 1, lora, out, opt->quant_layers,
                       opt->quant_type, {}, n, targets, false, quant_adapters);
    API_END
}

// Fills the empty adapter place `id` (the infer task's call, like bind_adapter); every refusal is decided on the host first
int32_t b200rwkv_load_adapter(b200rwkv_engine* e, int32_t id, const uint8_t* adapter_st, size_t adapter_len, float alpha) {
    API_BEGIN(e)
    REQUIRE(id >= 1, B200RWKV_ERR_INVALID, "load_adapter: id " + std::to_string(id) + " outside 1..n");
    REQUIRE(adapter_st && adapter_len > 8, B200RWKV_ERR_INVALID, "null adapter image");
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(id <= e->n_adapters, B200RWKV_ERR_INVALID, "load_adapter: id " + std::to_string(id) + " outside 1..n");
    std::lock_guard<std::mutex> lk(e->mu);
    REQUIRE(!e->place_full[id - 1], B200RWKV_ERR_STATE,
            "load_adapter: place " + std::to_string(id) + " holds an adapter (unload it first)");
    StFile f(adapter_st, adapter_len);
    check_adapter_files(e->model_shapes, {{&f, alpha}}, e->ad_quant_layers(), e->quant_type);
    for (auto& kv : f.tensors) {
        if (!ends_with(kv.first, ".lora.0")) continue;
        const std::string base = kv.first.substr(0, kv.first.size() - 7);
        bool planned = false;
        for (const b200rwkv_engine::AdMatrix& m : e->ad_mats) planned = planned || m.name == base;
        REQUIRE(planned, B200RWKV_ERR_UNSUPPORTED,
                "adapter on " + base + ": this engine holds no W' plan for it (its kind was not targeted at creation)");
    }
    e->load_place(id, f, alpha);
    API_END
}

// The refusals both weight updates share, on the host: the engine's kind, then each name against the model (known, listed
// once, the model's shape when the caller gives one) and its dtype against what creation accepts for that tensor
// (time_state: F16, BF16 or F32; any other tensor the build reads: F16; a tensor it does not read: anything).
static void check_update(const b200rwkv_engine* e, const std::vector<b200rwkv_engine::WeightIn>& in) {
    REQUIRE(e->world == 1 && !e->group, B200RWKV_ERR_UNSUPPORTED, "update_weights: tensor-parallel engines are not updated in place");
    REQUIRE(!e->had_loras, B200RWKV_ERR_UNSUPPORTED,
            "update_weights: this engine blended load-time LoRA files, which it no longer holds: create it again instead");
    std::set<std::string> seen;
    for (const b200rwkv_engine::WeightIn& w : in) {
        const StTensor* m = st_find(e->model_shapes, w.name);
        REQUIRE(m, B200RWKV_ERR_INVALID, "update_weights: the model has no tensor " + w.name);
        REQUIRE(seen.insert(w.name).second, B200RWKV_ERR_INVALID, "update_weights: " + w.name + " is listed twice");
        REQUIRE(!w.host || w.host->shape == m->shape, B200RWKV_ERR_INVALID, "update_weights: " + w.name + " differs in shape from the model's");
        const std::string dt = w.host ? w.host->dtype
                                      : w.dtype == B200RWKV_DTYPE_F16 ? "F16" : w.dtype == B200RWKV_DTYPE_BF16 ? "BF16" : "F32";
        auto it = e->fills.find(w.name);
        if (it == e->fills.end()) continue;
        const bool init = it->second.front().kind == FILL_INIT;
        if (w.host)
            REQUIRE(dt == "F16" || (init && (dt == "BF16" || dt == "F32")), B200RWKV_ERR_UNSUPPORTED,
                    "update_weights: tensor " + w.name + " is " + dt + (init ? ", expected F16 / F32 / BF16" : ", expected F16"));
    }
}

// New weights in place (the infer task's call, like load_adapter); every refusal is decided on the host first
int32_t b200rwkv_update_weights(b200rwkv_engine* e, const uint8_t* st, size_t len) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(st, B200RWKV_ERR_INVALID, "null image");
    StFile f(st, len);
    REQUIRE(!f.duplicate, B200RWKV_ERR_INVALID, "update_weights: the image names a tensor twice");
    REQUIRE(!f.tensors.empty(), B200RWKV_ERR_INVALID, "update_weights: the image holds no tensor");
    std::vector<b200rwkv_engine::WeightIn> in;
    for (auto& kv : f.tensors) in.push_back({kv.first, &kv.second, nullptr, B200RWKV_DTYPE_F16, kv.second.numel()});
    std::lock_guard<std::mutex> lk(e->mu);
    check_update(e, in);
    CK(cudaSetDevice(e->dev));
    struct Release { Buf<__half>& b; ~Release() { b = Buf<__half>(); } } release{e->d_tmp};
    e->fill_weights(in);
    API_END
}

int32_t b200rwkv_update_weights_device(b200rwkv_engine* e, int32_t n, const b200rwkv_weight_src* src) {
    API_BEGIN(e)
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(src, B200RWKV_ERR_INVALID, "null tensor table");
    REQUIRE(n >= 1, B200RWKV_ERR_INVALID, "update_weights_device: n must be >= 1");
    std::vector<b200rwkv_engine::WeightIn> in;
    for (int i = 0; i < n; ++i) {
        REQUIRE(src[i].name && src[i].data, B200RWKV_ERR_INVALID, "update_weights_device: null name or data in entry " + std::to_string(i));
        REQUIRE(src[i].dtype >= B200RWKV_DTYPE_F16 && src[i].dtype <= B200RWKV_DTYPE_F32, B200RWKV_ERR_INVALID,
                "update_weights_device: dtype of " + std::string(src[i].name) + " must be B200RWKV_DTYPE_F16, _BF16 or _F32");
        in.push_back({src[i].name, nullptr, src[i].data, src[i].dtype, 0});
    }
    std::lock_guard<std::mutex> lk(e->mu);
    check_update(e, in);
    for (b200rwkv_engine::WeightIn& w : in) w.numel = e->model_shapes.at(w.name).numel();
    CK(cudaSetDevice(e->dev));
    for (const b200rwkv_engine::WeightIn& w : in) {
        cudaPointerAttributes pa;
        CK(cudaPointerGetAttributes(&pa, w.dev));
        REQUIRE(pa.type == cudaMemoryTypeDevice && pa.device == e->dev, B200RWKV_ERR_INVALID,
                "update_weights_device: " + w.name + " is not memory of the engine's device");
    }
    struct Release { Buf<__half>& b; ~Release() { b = Buf<__half>(); } } release{e->d_tmp};
    e->fill_weights(in);
    API_END
}

// Empties adapter place `id` (the infer task's call); refused while a slot is bound to it
int32_t b200rwkv_unload_adapter(b200rwkv_engine* e, int32_t id) {
    API_BEGIN(e)
    REQUIRE(id >= 1, B200RWKV_ERR_INVALID, "unload_adapter: id " + std::to_string(id) + " outside 1..n");
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(id <= e->n_adapters, B200RWKV_ERR_INVALID, "unload_adapter: id " + std::to_string(id) + " outside 1..n");
    std::lock_guard<std::mutex> lk(e->mu);
    REQUIRE(e->place_full[id - 1], B200RWKV_ERR_STATE, "unload_adapter: place " + std::to_string(id) + " is empty");
    for (int s = 0; s < e->S; ++s)
        REQUIRE(e->slot_adapter[s] != id, B200RWKV_ERR_STATE,
                "unload_adapter: slot " + std::to_string(s) + " is bound to adapter " + std::to_string(id));
    e->unload_place(id);
    API_END
}

// Binds slots to adapters for the next infer calls (the infer task's call, like infer itself); every argument is checked
// before the table is touched
int32_t b200rwkv_bind_adapter(b200rwkv_engine* e, int32_t nslot, const int32_t* slots, const int32_t* adapter) {
    API_BEGIN(e)
    REQUIRE(slots && adapter, B200RWKV_ERR_INVALID, "bind_adapter: null list");
    REQUIRE(nslot >= 1 && nslot <= 1024, B200RWKV_ERR_INVALID, "bind_adapter: nslot must be in [1, max_batch]");
    for (int i = 0; i < nslot; ++i) {          // what needs no engine first
        REQUIRE(slots[i] >= 0, B200RWKV_ERR_STATE, "bind_adapter: slot out of range");
        REQUIRE(adapter[i] >= 0, B200RWKV_ERR_INVALID, "bind_adapter: unknown adapter id " + std::to_string(adapter[i]));
        for (int j = 0; j < i; ++j) REQUIRE(slots[j] != slots[i], B200RWKV_ERR_INVALID, "bind_adapter: duplicate slot");
    }
    REQUIRE(e, B200RWKV_ERR_INVALID, "null engine");
    REQUIRE(nslot <= e->S, B200RWKV_ERR_INVALID, "bind_adapter: nslot must be in [1, max_batch]");
    for (int i = 0; i < nslot; ++i) {
        REQUIRE(slots[i] < e->S, B200RWKV_ERR_STATE, "bind_adapter: slot out of range");
        REQUIRE(adapter[i] <= e->n_adapters, B200RWKV_ERR_INVALID, "bind_adapter: unknown adapter id " + std::to_string(adapter[i]));
    }
    std::lock_guard<std::mutex> lk(e->mu);
    for (int i = 0; i < nslot; ++i)
        REQUIRE(adapter[i] == 0 || e->place_full[adapter[i] - 1], B200RWKV_ERR_STATE,
                "bind_adapter: adapter place " + std::to_string(adapter[i]) + " is empty");
    for (int i = 0; i < nslot; ++i) e->slot_adapter[slots[i]] = adapter[i];
    if (e->n_adapters) {
        CK(cudaSetDevice(e->dev));
        CK(cudaMemcpyAsync(e->d_slot_adapter, e->slot_adapter.data(), (size_t)e->S * 4, cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));      // the step kernels read the table before griddepcontrol.wait
    }
    API_END
}

// One shrink launch on caller rows: x [T][K] f16 (precision 1: hi rows, then lo rows) packed into an A16 operand of K + 128 n
// columns, adapter b + 1 = lora_a[b] ([K][rank[b]] f16, as on disk), token t bound to ids[t]; tail <- the n tail blocks,
// [T][n][128] (precision 1: hi blocks, then lo blocks).  Tail cells start as NaN, so every cell the kernel misses shows.
int32_t b200rwkv_op_adapter(int32_t device, int32_t T, int32_t K, int32_t precision, int32_t n, const int32_t* rank,
                            const uint16_t* const* lora_a, const int32_t* ids, const uint16_t* x, uint16_t* tail) {
    API_BEGIN((b200rwkv_engine*)nullptr)
    REQUIRE(rank && lora_a && ids && x && tail, B200RWKV_ERR_INVALID, "null argument");
    REQUIRE(precision == 0 || precision == 1, B200RWKV_ERR_INVALID, "precision must be 0 or 1");
    REQUIRE(T >= 1 && T <= (precision ? 16 : A16_MAX_ROWS), B200RWKV_ERR_INVALID, "T must be 1..128 (1..16 with precision 1)");
    REQUIRE(K >= 8 && K % 8 == 0 && K <= 65536, B200RWKV_ERR_INVALID, "K must be a multiple of 8 in 8..65536");
    REQUIRE(n >= 1 && n <= AD_MAX, B200RWKV_ERR_INVALID, "n must be 1..8");
    for (int b = 0; b < n; ++b)
        REQUIRE(lora_a[b] && rank[b] >= 1 && rank[b] <= AD_MAX_RANK, B200RWKV_ERR_INVALID, "adapter matrix null or rank outside 1..128");
    for (int t = 0; t < T; ++t) REQUIRE(ids[t] >= 0 && ids[t] <= n, B200RWKV_ERR_INVALID, "adapter id outside 0..n");
    int ndev = 0;
    REQUIRE(cudaGetDeviceCount(&ndev) == cudaSuccess && device >= 0 && device < ndev, B200RWKV_ERR_CUDA, "no such CUDA device");
    CK(cudaSetDevice(device));
    const bool split = precision == 1;
    const int th = split ? 32 : 16 * mt_bucket(T), kb0 = cdiv(K, GEMM_BK);
    const size_t halves = (size_t)(kb0 + n) * A16_KB_HALVES;
    std::vector<uint16_t> op(halves, 0);
    for (int t = 0; t < T; ++t)
        for (int k = 0; k < K; ++k) {
            op[a16_index(t, k, th)] = x[(size_t)t * K + k];
            if (split) op[a16_index(t + 16, k, th)] = x[((size_t)T + t) * K + k];
        }
    for (int t = 0; t < (split ? 32 : T); ++t)
        for (int k = kb0 * GEMM_BK; k < (kb0 + n) * GEMM_BK; ++k) op[a16_index(t, k, th)] = 0x7E00;
    const int maxS = A16_MAX_ROWS;
    std::vector<int> meta(MetaView::ints(A16_MAX_ROWS, maxS), 0);
    MetaView hv{meta.data(), A16_MAX_ROWS, maxS};
    meta[0] = T; meta[1] = T;
    for (int t = 0; t < T; ++t) const_cast<int*>(hv.tok_slot())[t] = t;
    Buf<uint16_t> d_op(halves * 2);
    Buf<int> d_meta(meta.size() * 4), d_ids((size_t)T * 4);
    CK(cudaMemcpy(d_op, op.data(), halves * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_ids, ids, (size_t)T * 4, cudaMemcpyHostToDevice));
    std::vector<Buf<uint16_t>> d_a;
    AdapterParams P;
    memset(&P, 0, sizeof(P));
    P.nproj = 1; P.n = n; P.meta = MetaView{d_meta, A16_MAX_ROWS, maxS}; P.slot_adapter = d_ids; P.th = th;
    P.p[0].op = reinterpret_cast<__half*>((uint16_t*)d_op);
    P.p[0].K = K; P.p[0].kb0 = kb0;
    for (int b = 0; b < n; ++b) {
        const std::vector<uint16_t> rows = adapter_a_rows(reinterpret_cast<const uint8_t*>(lora_a[b]), K, rank[b]);
        d_a.emplace_back(rows.size() * 2);
        CK(cudaMemcpy(d_a.back(), rows.data(), rows.size() * 2, cudaMemcpyHostToDevice));
        P.p[0].A[b] = reinterpret_cast<const __half*>((uint16_t*)d_a.back());
        P.p[0].r[b] = rank[b];
    }
    if (split) adapter_shrink_kernel<true><<<adapter_grid(T, 1), AD_THREADS>>>(P);
    else adapter_shrink_kernel<false><<<adapter_grid(T, 1), AD_THREADS>>>(P);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(op.data(), d_op, halves * 2, cudaMemcpyDeviceToHost));
    for (int h = 0; h < (split ? 2 : 1); ++h)
        for (int t = 0; t < T; ++t)
            for (int b = 0; b < n; ++b)
                for (int j = 0; j < AD_MAX_RANK; ++j)
                    tail[(((size_t)h * T + t) * n + b) * AD_MAX_RANK + j] = op[a16_index(t + 16 * h, (kb0 + b) * GEMM_BK + j, th)];
    API_END
}

const char* b200rwkv_last_error(b200rwkv_engine* e) { (void)e; return g_err.c_str(); }

}  // extern "C"
