/* b200rwkv.h — C ABI of the H100-native RWKV inference engine.
 *
 * This is the drop-in boundary underneath crates/ai00-core: every entry point replaces one
 * use of the `web-rwkv` crate at a call site of the reference (paths relative to the
 * reference repository root).  The Rust shim that implements web-rwkv's `Runtime<Rnn>` /
 * `State` traits on top of these functions is given in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 on success, a negative b200rwkv_status on failure; the message
 *     of the calling thread's most recent failure is available from b200rwkv_last_error()
 *     (thread-local: the infer task and the softmax task never see each other's text).  No
 *     exception crosses the boundary.
 *   - all buffers are caller-owned plain host memory unless stated; nothing is retained after
 *     the call returns (the `.st` image is only borrowed during b200rwkv_create).
 *   - threading mirrors the reference: ONE task calls infer/state ops
 *     (crates/ai00-core/src/run.rs:1232) and ONE task calls softmax (run.rs:1237); the engine
 *     serialises each group with an internal mutex.
 *   - there is no CPU fallback: creation fails if no sm_90 (H100) device is present.
 */
#ifndef B200RWKV_H
#define B200RWKV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200rwkv_engine b200rwkv_engine;

typedef enum {
    B200RWKV_OK = 0,
    B200RWKV_ERR_INVALID = -1,     /* bad argument / malformed .st */
    B200RWKV_ERR_UNSUPPORTED = -2, /* model version or precision not supported */
    B200RWKV_ERR_CUDA = -3,        /* CUDA failure: the engine is dead, reload it */
    B200RWKV_ERR_STATE = -4        /* unknown slot / snapshot id */
} b200rwkv_status;

/* Mirror of web-rwkv `ModelInfo` as consumed at crates/ai00-core/src/lib.rs:587 and
 * crates/ai00-core/src/run.rs:672 (fields `version`, `num_vocab` are read by the core). */
typedef struct {
    int32_t version;            /* 5, 6 or 7 */
    int32_t num_layer;
    int32_t num_emb;
    int32_t num_hidden;
    int32_t num_vocab;
    int32_t num_head;
    int32_t head_size;
    int32_t time_mix_adapter;   /* v6 ddlerp LoRA rank */
    int32_t time_decay_adapter; /* v6 decay / v7 w LoRA rank */
} b200rwkv_info;

/* RnnOption (crates/ai00-core/src/run.rs:25, used at run.rs:710-724, 812-822). */
enum {
    B200RWKV_OPTION_LAST = 0,
    B200RWKV_OPTION_FULL = 1,
    /* consume the tokens, emit no logits: what a shim passes for a Last slot whose token run is
     * cut by token_chunk_size and continues in the next infer call (run.rs:1134-1145) */
    B200RWKV_OPTION_NONE = 2
};

/* Replaces `Loader::info(&SafeTensors)` — crates/ai00-core/src/lib.rs:587,
 * crates/ai00-server/src/api/file.rs:115.  Pure host code, no GPU needed. */
int32_t b200rwkv_info_from_st(const uint8_t* st, size_t len, b200rwkv_info* out);

/* Replaces `ModelBuilder::new(ctx, st).build_vN()` + `vN::Bundle::<f16>::new(model, max_batch)`
 * + `TokioRuntime::<Rnn>::new(bundle)` — crates/ai00-core/src/lib.rs:484-515.
 * `device` is the CUDA ordinal (the reference's adapter selection, lib.rs:351-368).
 * precision (the reference's `Precision`, lib.rs:493: `Bundle::<f16>` / `Bundle::<f32>` = the ACTIVATION type; weights
 * are f16 on disk and in HBM either way):
 *   0 = fp16: every projection input is rounded to f16 (tensor-core operand), f32 accumulate / state / logits;
 *   1 = fp32: no activation is rounded -- every projection input travels as an f16 hi + lo pair (two operand tiles,
 *       accumulators added), which is f32-exact to ~2^-22; steps are capped at 16 tokens. */
int32_t b200rwkv_create(const uint8_t* st, size_t len, int32_t device, int32_t max_batch,
                        int32_t token_chunk_size, int32_t precision, b200rwkv_engine** out);

/* Everything the reference's ReloadRequest carries for this path (crates/ai00-core/src/lib.rs:196-240, 484-497), one call:
 *   - devices: `num_devices` in {1, 2, 4, 8} CUDA ordinals of this box.  With more than one, the returned handle is ONE engine
 *     that owns every tensor-parallel rank (head / column parallel, SURVEY.md §8e) and one worker thread per rank: every call
 *     below is made once, by the same two tasks as before, and drives all GPUs -- the reference's single `Runtime` object
 *     (run.rs:1230-1234).  State tensors are merged / scattered by head inside state_back / state_load.
 *   - LoRA files blended into the projection matrices while they are uploaded (lib.rs:466-485, `LoraBlend::full(alpha)`):
 *     `<name>.lora.1` [out, r] and `<name>.lora.0` [in, r] as the reference's converter writes them
 *     (assets/scripts/convert_safetensors.py:96-101); W += alpha * lora.1 @ lora.0^T in f32, rounded once to f16.  Files with
 *     anything but low-rank pairs on att.{receptance,key,value,gate,output} / ffn.{key,value,receptance} / head are
 *     B200RWKV_ERR_UNSUPPORTED.  Images are borrowed during the call only.
 * Set struct_bytes = sizeof(b200rwkv_options); zero the rest for defaults (device 0, no LoRA, fp16). */
#define B200RWKV_MAX_LORA 4
typedef struct {
    uint32_t struct_bytes;
    int32_t max_batch, token_chunk_size, precision;
    int32_t num_devices;              /* 0 or 1: single GPU, devices[0] (0 if num_devices == 0) */
    int32_t devices[8];
    int32_t num_lora;
    const uint8_t* lora_st[B200RWKV_MAX_LORA];
    size_t lora_len[B200RWKV_MAX_LORA];
    float lora_alpha[B200RWKV_MAX_LORA];
    /* `quant` / `quant_type` of the reload request (lib.rs:211-215, 465: the first `quant_layers` layers keep their eight
     * projection matrices in a weight-only quantised format; everything else stays f16).  Single GPU, precision 0 only. */
    int32_t quant_layers;
    int32_t quant_type;               /* B200RWKV_QUANT_*: NONE, INT8, NF4, FP8 or INT4 (3 = SF4 and 5 are refused) */
    /* 1: batch-invariant engine.  Every per-token result of a slot (logits rows of LAST / FULL / snapshots, SCORE values and
     * argmax ids, the kept row, the state after every token, recorded and pooled hidden rows) is then a function of the
     * model, the precision, the slot's starting state and the tokens it has fed only: bit-identical whatever the other
     * entries of the call are, whatever token_chunk_size is and however the tokens are cut into calls.  The reference is
     * the decode step (one token per entry, at most 16 entries): steps of more than 16 tokens run each token with its
     * arithmetic (DESIGN.md §6, batch-invariant engines).  0: off (the default; nothing changes).  Any other value is
     * B200RWKV_ERR_INVALID; 1 with num_devices > 1, or with b200rwkv_create_adapters / b200rwkv_create_adapter_places, is
     * B200RWKV_ERR_UNSUPPORTED (all before any CUDA call).  With precision 1 the flag is accepted and changes nothing: those steps are capped at 16
     * tokens and already decode-shaped.  struct_bytes = offsetof(b200rwkv_options, batch_invariant), the size before this
     * field, is accepted and means 0. */
    int32_t batch_invariant;
    /* 1: adapters (b200rwkv_create_adapters, b200rwkv_create_adapter_places, b200rwkv_load_adapter) may pair matrices of the
     * quantised layers, and a places engine's `targets` also plan the targeted kinds there.  For a token bound to adapter a,
     * such a projection computes  act(x Wq^T + f16(alpha_a B_a) r(x A_a^T) + bias)  with Wq the format's dequantised matrix
     * (B200RWKV_QUANT_*); the adapter term is not scaled by an FP8 row scale, and the adapter matrices are never quantised.
     * Resident memory: the quantised W' plans hold the layer's codes a second time, plus one f16 128-wide tail block per place.
     * 0: off (the default; such pairs are B200RWKV_ERR_UNSUPPORTED).  Any other value is B200RWKV_ERR_INVALID; 1 with
     * num_devices > 1 is B200RWKV_ERR_UNSUPPORTED (both before any CUDA call).  With b200rwkv_create_ex, or with
     * quant_layers 0, the flag is accepted and changes nothing.  The field fills the struct's tail padding, so sizeof is
     * unchanged and a caller who zeroed the struct reads 0; struct_bytes = offsetof(b200rwkv_options, batch_invariant) means 0
     * too. */
    int32_t quant_adapters;
} b200rwkv_options;
#define B200RWKV_QUANT_NONE 0
#define B200RWKV_QUANT_INT8 1         /* blocks of 128 inputs: f16 (min, max) + 8-bit codes */
#define B200RWKV_QUANT_NF4 2          /* blocks of 64 inputs: f16 absmax + 4-bit NormalFloat codes */
                                      /* Quant::SF4 is not implemented: create_ex answers B200RWKV_ERR_UNSUPPORTED */
#define B200RWKV_QUANT_FP8 4          /* beyond the reference's Quant enum: E4M3 codes, one f32 scale max|w| / 448 per output row
                                       * of the whole matrix; the projection multiplies the codes' exact values with the f16
                                       * operand in f32 and scales each output.  Same refusals as Int8 / NF4 (one GPU,
                                       * precision 0, no adapters on its layers unless quant_adapters); batch-invariant
                                       * engines run it. */
#define B200RWKV_QUANT_INT4 6         /* beyond the reference's Quant enum: Int8's scheme at 4 bits.  Blocks of 128 inputs of one
                                       * output row keep scale = f16((max - min) / 15), min = f16(min) and 4-bit codes
                                       * q = floor(15 (w - min) / (max - min) + 0.5); the projection multiplies
                                       * fma_f16(q, scale, min) (one rounding) with the f16 operand in f32.  Same refusals as
                                       * Int8 / NF4 (one GPU, precision 0, no adapters on its layers unless quant_adapters);
                                       * batch-invariant engines run it. */
int32_t b200rwkv_create_ex(const uint8_t* st, size_t len, const b200rwkv_options* opt, b200rwkv_engine** out);

/* Several LoRA adapters on one resident base model, chosen per slot at run time (the reference can only blend LoRA files at
 * load and needs a restart to drop one, docs/doc-guide/features.md).
 * b200rwkv_create_adapters = b200rwkv_create_ex plus n (1..8) adapter files kept unblended on the device, ids 1..n.  Adapter
 * files have the load-time LoRA format: `<name>.lora.0` [in, r] and `<name>.lora.1` [out, r], F16, pairs only on
 * att.{receptance,key,value,gate,output}, ffn.{key,value,receptance} and head; full tensors and unknown targets are
 * B200RWKV_ERR_UNSUPPORTED, a missing half or a shape that does not match the matrix B200RWKV_ERR_INVALID, a rank above 128
 * B200RWKV_ERR_UNSUPPORTED.  Also B200RWKV_ERR_UNSUPPORTED: more than one device, and a pair on a matrix of a quantised layer
 * (opt->quant_layers) unless opt->quant_adapters.  All of this is checked before any CUDA call.  Images are borrowed during the call only.  LoRA files in
 * `opt` are blended into the base first; adapters apply on top of them.
 * Meaning: for a token whose slot is bound to adapter a, every projection W with a pair in a computes
 *   act(x W^T + u B'^T + bias),  u = x A^T (A = lora.0^T) rounded like the operand x (f16, or an f16 hi + lo pair with
 *   precision 1),  B' = f16(alpha_a * lora.1)
 * -- the unblended form of create_ex with lora = [(file_a, alpha_a)].
 * b200rwkv_bind_adapter: slot slots[i] runs adapter[i] (0 = the base model) from the next infer call on.  A binding belongs to
 * the slot, not to its state: state_load / state_write / snapshots and the kept row neither carry nor clear it (a kept row is
 * what the slot's last LAST / FULL / SCORE entry computed, under the adapter bound then).  Called by the infer task, like
 * b200rwkv_infer.  Checked before any CUDA call: nslot outside [1, max_batch], a duplicate slot or an adapter id outside
 * 0..n is B200RWKV_ERR_INVALID, a slot out of range B200RWKV_ERR_STATE.  On engines from the other constructors only id 0
 * exists.  Slots bound to different adapters and unbound slots mix freely in one call; a step in which no slot is bound runs
 * exactly the launches (and gives exactly the bits) of a create_ex engine.
 * Resident memory: every projection launch an adapter touches is held a second time, with one 128-wide k block per adapter
 * appended (W' = [W | alpha_1 B_1 | ...]), plus each adapter's A matrices; adapters on every projection kind and the head cost
 * about the projection weights again (7B: +14.7 GB, + 1.5 GB of tail blocks and 1.4 GB of A for 4 adapters: A is reserved at
 * rank 128, so that b200rwkv_unload_adapter / b200rwkv_load_adapter below can replace a file by one of any rank). */
int32_t b200rwkv_create_adapters(const uint8_t* st, size_t len, const b200rwkv_options* opt, int32_t n,
                                 const uint8_t* const* adapter_st, const size_t* adapter_len, const float* adapter_alpha,
                                 b200rwkv_engine** out);
int32_t b200rwkv_bind_adapter(b200rwkv_engine*, int32_t nslot, const int32_t* slots, const int32_t* adapter);

/* Adapters that come and go while the engine serves (the reference fixes its LoRA files at load; dropping one means a restart).
 * b200rwkv_create_adapter_places = b200rwkv_create_ex plus n (1..8) empty adapter places, ids 1..n.  A place can hold an
 * adapter file with pairs on the `targets` kinds of matrix (B200RWKV_TARGET_* bits) in every layer that is not quantised
 * (opt->quant_layers; every layer with opt->quant_adapters), and on the head if targeted; bits for matrices the model does not have (ATT_G, FFN_R on v7) are
 * skipped.  Refused before any CUDA call: n outside 1..8, targets 0 or an unknown bit, a NULL out / opt or a wrong
 * struct_bytes are B200RWKV_ERR_INVALID; more than one device, or targets that name no f16 matrix of the model,
 * B200RWKV_ERR_UNSUPPORTED.
 * b200rwkv_load_adapter fills the empty place `id` with an adapter file (the format of b200rwkv_create_adapters).  Afterwards
 * slots bound to `id` compute exactly what they would on an engine made by b200rwkv_create_adapters with that file at that
 * id, under the same plans.  Refused, with nothing changed and before any CUDA call: id outside 1..n, a NULL image, a missing
 * half or a shape that does not match its matrix are B200RWKV_ERR_INVALID; a place that holds an adapter B200RWKV_ERR_STATE
 * (replacing one is an unload, then a load, so a bound slot never changes adapter silently); full tensors, non-F16 pairs, a
 * rank above 128, a pair on a quantised layer (unless quant_adapters) and a pair on a matrix this engine holds no W' plan for are
 * B200RWKV_ERR_UNSUPPORTED.  The plans: on a places engine every targeted matrix of the f16 layers; on a
 * b200rwkv_create_adapters engine the matrices its files paired at creation (its n places start full).
 * b200rwkv_unload_adapter empties place `id`: id outside 1..n is B200RWKV_ERR_INVALID; an empty place, or one a slot is bound
 * to, B200RWKV_ERR_STATE (the message names the slot).  b200rwkv_bind_adapter to an empty place is B200RWKV_ERR_STATE.
 * All three are made by the infer task, like bind_adapter.  Their writes go on the engine's stream, so steps already enqueued
 * finish with the old contents, and are complete when the call returns; the image is only borrowed.  Slots bound to other
 * places, unbound slots, states, kept rows and snapshots are not touched.  The captured step graphs of bound steps are
 * dropped and captured again on their next use; unbound steps keep theirs.
 * Resident memory is reserved at creation (load_adapter allocates none).  Figures computed from shapes, not measured, for the
 * 7B shape (C = 4096, F = 14336, L = 32, V = 65536) with every kind and the head targeted:
 *   - W' plans: about the projection bytes again, +14.7 GB;
 *   - one 128-wide tail column per place on every planned matrix: 128 * (7 C + F) * 2 B * L + 128 * V * 2 B, about
 *     0.37 GB per place;
 *   - A rows for rank 128 per place and planned matrix: 128 * (5 C + 2 C + F) * 2 B * L + 128 * C * 2 B, about 0.35 GB
 *     (0.33 GiB) per place (b200rwkv_create_adapters engines reserve the same, so a place can be reloaded with any rank).
 * Step cost: a step with a bound slot streams the tail blocks of all n places, full or empty -- the cost of a
 * b200rwkv_create_adapters engine with n files.  Size n to what is needed. */
#define B200RWKV_TARGET_ATT_R  (1u << 0)   /* att.receptance */
#define B200RWKV_TARGET_ATT_K  (1u << 1)   /* att.key */
#define B200RWKV_TARGET_ATT_V  (1u << 2)   /* att.value */
#define B200RWKV_TARGET_ATT_G  (1u << 3)   /* att.gate (v5 / v6) */
#define B200RWKV_TARGET_ATT_O  (1u << 4)   /* att.output */
#define B200RWKV_TARGET_FFN_K  (1u << 5)   /* ffn.key */
#define B200RWKV_TARGET_FFN_V  (1u << 6)   /* ffn.value */
#define B200RWKV_TARGET_FFN_R  (1u << 7)   /* ffn.receptance (v5 / v6) */
#define B200RWKV_TARGET_HEAD   (1u << 8)
int32_t b200rwkv_create_adapter_places(const uint8_t* st, size_t len, const b200rwkv_options* opt, int32_t n,
                                       uint32_t targets, b200rwkv_engine** out);
int32_t b200rwkv_load_adapter(b200rwkv_engine*, int32_t id, const uint8_t* adapter_st, size_t adapter_len, float alpha);
int32_t b200rwkv_unload_adapter(b200rwkv_engine*, int32_t id);

/* New weights for a live engine, in place: a trainer's next iterate, or a same-shape fine-tune, without destroying the
 * engine and creating it again.  Afterwards the engine computes, bit for bit, what an engine created now would compute with
 * the same options and constructor, the same adapter files (for places: the same files loaded at the same ids), and the
 * model image with the listed tensors replaced: logits rows, states, SCORE values and argmax ids, score_top lists, kept and
 * pooled hidden rows, sample_topk / sample_probs results, and launch counts.
 * b200rwkv_update_weights takes a safetensors image holding any subset of the model's tensors; the rest keep their values.
 * b200rwkv_update_weights_device takes n tensors already on the engine's device, each dense in the model's shape: F16, BF16
 * or F32, rounded to F16 (round to nearest even) by a conversion kernel, so the result is that of update_weights with an
 * image of the rounded values.  time_state is read as f32 from any of the three, as creation reads it.
 * Everything the build derives from a listed tensor is derived again by the build's own kernels: repacked f16 blocks,
 * Int8 / NF4 / FP8 / Int4 codes and scales (an FP8 row scale over the whole row, split-K slices included), the base part of
 * every W' plan, f32 vectors, the v5 decay table, the v6 k-major time_decay_w2 copy, the embedding, the head, and State::init
 * (b200rwkv_state_init) from time_state.  Left alone: adapter tail blocks and A rows, adapter bindings, keep_hidden* and
 * score_top settings, the captured step graphs (every weight buffer stays where it is), and slot states, snapshots and kept
 * logits rows: those still hold what the OLD weights computed.  Dropping or recomputing them is the caller's decision; a
 * rollout loop drops its cached states after every update (INTEGRATION.md §8).
 * Refused, before any CUDA call and with nothing changed: a NULL engine, image or table, n < 1, a malformed image, a name
 * the model does not have, a name listed twice, a shape that differs from the model's, or a device dtype other than the three
 * are B200RWKV_ERR_INVALID; a dtype creation refuses for that tensor (an image's matrix in BF16, say), an engine created with
 * load-time LoRA files (opt->lora_st: their images were only borrowed, so the blend cannot be redone) and a tensor-parallel
 * engine are B200RWKV_ERR_UNSUPPORTED.  A device pointer that is not memory of the engine's device is B200RWKV_ERR_INVALID.
 * Made by the infer task, like load_adapter.  The writes go on the engine's stream, so steps already enqueued finish with the
 * old weights, and are complete when the call returns.  The call holds a staging buffer the size of its largest tensor (as
 * creation does) and allocates no resident memory.  An image from b200rwkv_host_alloc (pinned) uploads faster than pageable
 * memory (DESIGN.md §6). */
int32_t b200rwkv_update_weights(b200rwkv_engine*, const uint8_t* st, size_t len);
#define B200RWKV_DTYPE_F16  0
#define B200RWKV_DTYPE_BF16 1
#define B200RWKV_DTYPE_F32  2
typedef struct {
    const char* name;       /* the model's tensor name, e.g. "blocks.3.att.key.weight" */
    int32_t dtype;          /* B200RWKV_DTYPE_* */
    const void* data;       /* device pointer on the engine's device, dense, the model's shape */
} b200rwkv_weight_src;
int32_t b200rwkv_update_weights_device(b200rwkv_engine*, int32_t n, const b200rwkv_weight_src* src);

/* The vocabulary head's weight format from the next infer call on.  quant_type: B200RWKV_QUANT_NONE (f16, the default), INT8,
 * NF4, FP8 or INT4 -- the quantiser and block layout of quantised layers, applied to head.weight.  The head is the one matrix
 * every decode step streams whole; once the layers are quantised it is a large share of the step's bytes (DESIGN.md §4a).
 *   - Meaning: every head launch computes logits = x Wq^T, Wq the format's dequantised head.weight (Int8 / Int4: blocks of
 *     128 inputs, NF4: blocks of 64, FP8: one f32 scale per vocabulary row, which multiplies x Wq^T as in the layer kernels),
 *     x the unchanged f16 operand.  That is the step's head launch, the snapshot rows' head launch, the head launch of steps
 *     with bound adapter slots, bench_decode, profile_step, profile_insitu and debug_gemm_time(which = 30).  SCORE,
 *     score_top, sample_topk, sample_probs, kept rows and hidden rows read the rows the head wrote, unchanged.
 *   - The codes are those b200rwkv_op_quantize gives for head.weight as creation saw it (LoRA files blended in), quantised on
 *     the device from the resident f16 head.  b200rwkv_update_weights / _device with head.weight derive them again, so the
 *     result is bit-identical to a new engine from the new image with the same head format.
 *   - NONE returns to the f16 head bit for bit: rows, states and launch counts equal those of an engine that never called
 *     this.  Setting the current format again does nothing.  Slot states, snapshots and kept rows are left as they are and
 *     hold what the old head computed.  A quantised head launches exactly as many kernels as the f16 head.
 *   - Memory: the f16 head stays resident.  The call allocates the codes (7B head, V = 65536, C = 4096: FP8 0.27 GB, Int8
 *     0.28 GB, Int4 and NF4 0.14 GB) and releases those of the previous format; while it runs it also holds a staging
 *     buffer the size of the f16 head.  If an allocation fails the call fails with the previous head in place.
 *   - Made by the infer task, like update_weights.  The writes go on the engine's stream, so steps already enqueued finish
 *     with the old head; the captured step graphs are dropped and captured again on their next use.
 *   - Refused before any CUDA call, with nothing changed: a NULL engine or a value outside 0..6 is B200RWKV_ERR_INVALID;
 *     3 (SF4) and 5, a tensor-parallel engine (either front end), precision 1, num_emb not a multiple of 128, and an engine
 *     whose adapters plan the head (a b200rwkv_create_adapters file with a head pair, or places with B200RWKV_TARGET_HEAD)
 *     are B200RWKV_ERR_UNSUPPORTED.  Batch-invariant engines keep their guarantee with a quantised head. */
int32_t b200rwkv_head_format(b200rwkv_engine*, int32_t quant_type);

/* Tensor-parallel construction, one process per GPU (head / column parallel, SURVEY.md §8e).
 * (The in-process alternative -- one handle, all ranks inside -- is b200rwkv_create_ex above.)
 * Every rank calls create_tp with the same model, then exchanges the opaque handle blobs
 * (b200rwkv_tp_export on each rank, all-gathered by the host over any side channel) and
 * passes all `world` blobs, rank-ordered, to b200rwkv_tp_connect.  After that every API call
 * is SPMD: all ranks make the same call with the same arguments.  Rank 0 receives the full
 * [rows, num_vocab] logits (gathered from every rank's vocabulary shard over NVLink peer
 * memory); the other ranks' logits_out may be NULL.  State tensors are sharded by head:
 * state_back on rank r fills the WKV rows of its own heads and zeros elsewhere. */
#define B200RWKV_TP_HANDLE_BYTES 128
int32_t b200rwkv_create_tp(const uint8_t* st, size_t len, int32_t device, int32_t max_batch,
                           int32_t token_chunk_size, int32_t precision, int32_t rank, int32_t world,
                           b200rwkv_engine** out);
int32_t b200rwkv_tp_export(b200rwkv_engine*, uint8_t handle_out[B200RWKV_TP_HANDLE_BYTES]);
int32_t b200rwkv_tp_connect(b200rwkv_engine*, const uint8_t* handles /* world * HANDLE_BYTES */);
/* Same wiring when all ranks live in one process (rank-ordered array of engines). */
int32_t b200rwkv_tp_connect_local(b200rwkv_engine** engines, int32_t n);

/* Dropping the `Arc<dyn Runtime>` (crates/ai00-core/src/lib.rs:600,654). */
void b200rwkv_destroy(b200rwkv_engine*);

int32_t b200rwkv_get_info(b200rwkv_engine*, b200rwkv_info* out);

/* Replaces `Runtime::infer(RnnInput)` — crates/ai00-core/src/run.rs:1143 — for one
 * `RnnInput`: a ragged batch of `nslot` entries; entry i feeds `ntok[i]` tokens
 * (tokens + sum(ntok[0..i])) to state slot `slot[i]` with RnnOption `option[i]`.
 * All tokens are consumed (internally in steps of at most min(token_chunk_size, 128) tokens shared evenly over the
 * entries, the policy
 * web-rwkv applies across calls at run.rs:1134-1145).  Logits rows (num_vocab f32 each) are
 * written contiguously to `logits_out` in entry order: 1 row for LAST (0 if ntok[i]==0),
 * ntok[i] rows for FULL, none for NONE; rows_out[i] receives the row count of entry i
 * (== RnnOutputBatch being empty or not, run.rs:1146-1155).  `logits_cap` is in floats.
 * `logits_out` may be NULL: nothing is copied to the host, the last row of every slot stays in HBM for
 * b200rwkv_sample_topk / b200rwkv_sample_probs.  Token ids >= num_vocab are B200RWKV_ERR_INVALID.
 * The slot's kept row: a LAST entry with tokens, a FULL or a SCORE entry makes the entry's last row the slot's kept row; a
 * NONE entry with tokens advances the state without a row and drops the kept row (the slot has none until its next LAST /
 * FULL / SCORE entry or b200rwkv_state_write); an entry with ntok = 0 leaves the kept row as it was. */
int32_t b200rwkv_infer(b200rwkv_engine*, int32_t nslot, const int32_t* slot, const int32_t* ntok,
                       const uint32_t* tokens, const int32_t* option, float* logits_out,
                       size_t logits_cap, int32_t* rows_out);

/* b200rwkv_infer plus scoring on the device: what the reference's perplexity() and choose path (run.rs:699-755, 936-983)
 * compute from RnnOption::Full rows, without moving those rows to the host.  A SCORE entry i with tokens x_0 .. x_{n-1}:
 *   - consumes its tokens as FULL does: the slot's state and kept row (the last row, what b200rwkv_sample_topk reads) are
 *     bit-identical to the same call with FULL;
 *   - rows_out[i] = 0: no logits row goes to `logits_out`;
 *   - score_out[j] = log softmax(row predicting x_j)[x_j] in f32, computed as (x_t - m) - logf(sum expf(x - m)), m the row
 *     maximum; the row predicting x_j is the row after x_{j-1} for j >= 1, and the slot's kept row for j = 0 (the row of the
 *     slot's current state: from the previous infer call, or from b200rwkv_state_write of a snapshot that carries a row;
 *     none, as after b200rwkv_state_load or a NONE entry with tokens: NaN);
 *   - argmax_out[j] = id of the largest logit of that row, lowest id on ties (UINT32_MAX if there is no row);
 *   - special values: a NaN anywhere in the row makes score_out[j] NaN, and argmax_out[j] is the lowest id of the largest
 *     non-NaN logit (UINT32_MAX if every logit is NaN); a -inf target in a row with a finite maximum scores -inf; a row of
 *     only -inf scores NaN with argmax 0; a target so far below the maximum that x_t - m overflows f32 scores -inf.
 * score_out / argmax_out hold sum(ntok) over the SCORE entries, in entry order; argmax_out may be NULL.  LAST, FULL, NONE and
 * SCORE entries mix freely in one call.  Every argument is checked before the first CUDA call.  Tensor parallel engines answer
 * B200RWKV_ERR_UNSUPPORTED for SCORE entries.  b200rwkv_infer refuses option 3. */
#define B200RWKV_OPTION_SCORE 3
typedef struct {
    uint32_t struct_bytes;          /* = sizeof(b200rwkv_infer_args) */
    int32_t nslot;
    const int32_t *slot, *ntok;
    const uint32_t* tokens;
    const int32_t* option;
    float* logits_out;              /* exactly as b200rwkv_infer */
    size_t logits_cap;
    int32_t* rows_out;
    float* score_out;               /* [sum of ntok over SCORE entries], entry order */
    uint32_t* argmax_out;           /* same shape, may be NULL */
} b200rwkv_infer_args;
int32_t b200rwkv_infer_ex(b200rwkv_engine*, const b200rwkv_infer_args* args);

/* `State` trait object — crates/ai00-core/src/lib.rs:399,494; uses at run.rs:477,1099-1107.
 * The host-visible state of one slot is an f32 tensor of web-rwkv shape [C, N+2, L, 1]
 * (x fastest; run.rs:987): row 0 time-mix shift, rows 1..N WKV, row N+1 channel-mix shift. */
int32_t b200rwkv_state_shape(b200rwkv_engine*, int64_t shape[4]);
int32_t b200rwkv_state_init(b200rwkv_engine*, float* out);                          /* State::init  */
/* State::load drops the slot's kept logits row: a host state carries none.  State::write makes the snapshot's row (or none,
 * if the snapshot has none) the slot's kept row; State::read takes the kept row into the snapshot. */
int32_t b200rwkv_state_load(b200rwkv_engine*, int32_t slot, const float* in);        /* State::load  */
int32_t b200rwkv_state_back(b200rwkv_engine*, int32_t slot, float* out);             /* State::back  */
int32_t b200rwkv_state_read(b200rwkv_engine*, int32_t slot, uint64_t* snapshot_id);  /* State::read  (device copy) */
int32_t b200rwkv_state_write(b200rwkv_engine*, int32_t slot, uint64_t snapshot_id);  /* State::write */
int32_t b200rwkv_state_free(b200rwkv_engine*, uint64_t snapshot_id);                 /* drop TensorGpu */

/* b200rwkv_infer_ex(args), and also snapshot k of the state of entry snap_entry[k]'s slot after the first snap_tokens[k]
 * tokens that entry feeds in this call (1 <= snap_tokens[k] <= ntok[entry]): what b200rwkv_state_read would have returned
 * had the call ended there, for a prefix-cache item at a shared boundary or a rollback after verifying several tokens.
 *  - A snapshot always carries the logits row of its token (the row predicting the next token), whatever the entry's
 *    option.  It is bit-identical to that token's logits_out row (FULL), the row its SCORE entry scored against, or, at a
 *    LAST entry's last token, the slot's kept row.  Other rows come from a head launch of their own.
 *  - snap_ids[k] is in / out: 0 asks for a new snapshot, whose id is written back; an existing id is overwritten in place,
 *    state and row, with no new state allocation (an id that had no row gains one).
 *  - Every other output is bit-identical to the same infer_ex call: logits_out, rows_out, scores, argmax ids, the slots'
 *    states, kept rows and recorded or pooled hidden rows.  Snapshot rows never reach logits_out or a kept row.  With
 *    nsnap == 0 the call launches exactly what infer_ex launches.
 *  - The step packing is infer_ex's.  A step that holds snapshots runs the same launches with their snapshot variants
 *    (the LN stages, WKV and ln_out also write the snapshot tokens' state), plus 1 row copy launch, plus, when one of its
 *    snapshot tokens has no output row (mid-run LAST / NONE, or NONE at the end), 1 head launch over those tokens (and 1
 *    adapter shrink launch in front of it when a slot of the step is bound to an adapter and any adapter of the engine has a
 *    pair on the head: the shrink the step's main head launch runs as well).  A
 *    snapshot does not carry an adapter binding, as with state_read.
 *  - Bytes per snapshot: L * (2C + H * 64 * 64) * 4 of state plus num_vocab * 4 of logits row: 34.6 MB of state at the 7B
 *    shape, 21.6 MB at 3B / v7-2b9.
 *  - Refused before any CUDA call, with nothing changed: everything infer_ex refuses; B200RWKV_ERR_INVALID for nsnap < 0,
 *    NULL arrays with nsnap > 0, an entry index outside [0, nslot), a position outside [1, ntok], a duplicate (entry,
 *    position) or one nonzero id listed twice; B200RWKV_ERR_STATE for an unknown nonzero id; B200RWKV_ERR_UNSUPPORTED
 *    for nsnap > 0 under tensor parallelism (either front end; nsnap == 0 runs as infer_ex there too). */
int32_t b200rwkv_infer_snapshots(b200rwkv_engine*, const b200rwkv_infer_args* args, int32_t nsnap, const int32_t* snap_entry,
                                 const int32_t* snap_tokens, uint64_t* snap_ids);

/* Device-resident state cache (SURVEY.md §8f-4).  The reference's cache holds `CachedItem { state: TensorCpu, output:
 * TensorCpu }` (crates/ai00-core/src/run.rs:199-205): every check-out / check-in is a State::load / State::back PCIe copy of
 * the whole state (34.6 MB per slot at 7B; run.rs:838, 996, 561).  Here a cached item is a snapshot id: state_read /
 * state_write are device-to-device copies, and the snapshot carries the slot's last logits row with it, so a cache hit can
 * be sampled on the device (b200rwkv_sample_topk) without re-running a token.  The two calls below move a snapshot to / from
 * host tensors without occupying a slot -- for spilling under memory pressure (b200rwkv_cache_stats), for `InputState::Value`
 * / `.state` files (run.rs:390-437) and for `/api/oai/states` (run.rs:984-989).  state: [C, N+2, L, 1] f32 as in
 * b200rwkv_state_back; logits: [num_vocab] f32, either pointer may be NULL (logits_out: ERR_STATE if the snapshot has no row). */
int32_t b200rwkv_snapshot_back(b200rwkv_engine*, uint64_t snapshot_id, float* state_out, float* logits_out);
int32_t b200rwkv_snapshot_load(b200rwkv_engine*, const float* state_in, const float* logits_in, uint64_t* snapshot_id);
int32_t b200rwkv_cache_stats(b200rwkv_engine*, int64_t* num_snapshots, int64_t* bytes_used, int64_t* bytes_free);

/* Replaces `vN::read_state(&context, &info, reader)` — crates/ai00-core/src/lib.rs:378-389 (initial states of state-tuned
 * models and `.state` files, run.rs:403-437): reads `blocks.{l}.att.time_state` [H, N, N] (F16 / F32 / BF16; the layout the
 * converter writes, crates/converter/src/main.rs:20) into the state tensor `out` ([C, N+2, L, 1] f32).  Host only. */
int32_t b200rwkv_read_state(const b200rwkv_info* info, const uint8_t* st, size_t len, float* out);

/* Replaces `web_rwkv::runtime::softmax::softmax(&context, Vec<TensorCpu<f32>>)` —
 * crates/ai00-core/src/run.rs:1179.  in/out: [rows, num_vocab] f32.  out = expf(x - max) * (1 / sum expf(x - max)) per row,
 * in f32; a -inf entry gives exactly 0.  Every row needs at least one finite entry (a row of only -inf is NaN); NaN inputs
 * are outside the contract. */
int32_t b200rwkv_softmax(b200rwkv_engine*, int32_t rows, const float* in, float* out);

/* GPU front half of token sampling (SURVEY.md §8f-1).  Replaces, for samplers that only need the head of the sorted
 * distribution (Nucleus with top_k <= 128 -- the reference default, sampler/nucleus.rs:16-17 -- and greedy), the per-token
 * per-slot sequence of crates/ai00-core/src/run.rs:664-697: `output.to_vec()` (num_vocab f32 D2H), `Sampler::transform`
 * (penalties, sampler/nucleus.rs:61-67), `Formatter::transform` (BNF mask, sampler/bnf.rs:37-40), the bias add
 * (run.rs:679-681), the softmax round trip (run.rs:1164-1190) and the full-vocabulary sort of
 * sampler/nucleus.rs:69-80.  Pass `logits_out = NULL` to b200rwkv_infer: the logits stay in HBM, and this call returns, for
 * each listed slot, the `top_k` most probable tokens of that slot's kept logits row (the row of its current state, see
 * b200rwkv_infer; a slot without one, as after b200rwkv_state_load or a NONE entry with tokens, is B200RWKV_ERR_STATE) after
 *     logits[penalty_token[j]] -= penalty_value[j]     j in [penalty_offset[i], penalty_offset[i+1])
 *     logits[t] = -inf  where bit t of allow_bits row i is 0                    (allow_bits may be NULL)
 *     logits[bias_token[j]]    += bias_value[j]        j in [bias_offset[i], bias_offset[i+1])
 * (tokens distinct within one row's penalty list and within its bias list, as the reference's HashMaps are), with
 * probs = softmax over the whole adjusted row.  Order: logit descending, token id ascending on ties.  ids_out / probs_out:
 * [nrows][top_k].  The draw itself (top_p cut, temperature, RNG, penalty update; nucleus.rs:81-123) stays in the host
 * sampler, now over <= 128 pairs.  Samplers that need the whole distribution (Mirostat, Typical, Nucleus with top_k > 128)
 * use b200rwkv_sample_probs below.  A row whose every token is disallowed yields ids 0 .. top_k-1, each with probability 0;
 * more generally, after the tokens with a finite adjusted logit come the lowest disallowed ids, in ascending order.
 * Penalty and bias tokens >= num_vocab are ignored.  top_k outside [1, min(128, num_vocab)] is B200RWKV_ERR_INVALID, checked
 * before any CUDA call.  Thread contract: the softmax task's (run.rs:1237). */
int32_t b200rwkv_sample_topk(b200rwkv_engine*, int32_t nrows, const int32_t* slots, const int32_t* penalty_offset,
                             const uint32_t* penalty_token, const float* penalty_value, const uint32_t* allow_bits,
                             const int32_t* bias_offset, const uint32_t* bias_token, const float* bias_value, int32_t top_k,
                             uint32_t* ids_out, float* probs_out);

/* The whole adjusted distribution on the device, for samplers that read every probability: MirostatSampler
 * (sampler/mirostat.rs:44-90), TypicalSampler (sampler/typical.rs:70-131) and NucleusSampler with top_k > 128.  Writes, for
 * each listed slot's kept logits row (the row of its current state, the row b200rwkv_sample_topk reads), exactly the vector
 * run.rs:673-691 hands to `Sampler::sample`: probs_out[i] = softmax(row adjusted as in b200rwkv_sample_topk), [nrows][num_vocab] f32, the adjustment
 * lists meaning and validated what they do there (allow_bits may be NULL).  The sampler itself stays on the host, unchanged.
 *   - probabilities are expf(x - max) * (1 / sum expf(x - max)) in f32; a disallowed token is exactly 0.  For num_vocab <=
 *     65536 every candidate probability b200rwkv_sample_topk returns for the same row and lists equals probs_out[i][id].
 *   - a row whose every token is disallowed is all zeros, as b200rwkv_sample_topk's probabilities are on such a row.
 *   - any num_vocab.  A row's result depends neither on which other rows the call lists nor on their order.
 *   - every argument is checked before the first CUDA call: nrows outside [1, max_batch], NULL slots / probs_out, a duplicate
 *     slot or bad adjustment lists are B200RWKV_ERR_INVALID; a slot out of range or without a kept row is B200RWKV_ERR_STATE.
 *   - the kept rows are not modified.  Tensor parallel engines run it on rank 0, which holds the gathered rows.
 * With b200rwkv_infer(logits_out = NULL) first, one num_vocab f32 row per slot crosses PCIe per token (256 KiB at 65536)
 * instead of a logits copy, an upload of the adjusted row and a probabilities copy.  probs_out may be any host memory; pinned
 * memory (b200rwkv_host_alloc) makes that copy about 4x faster (DESIGN.md §6).  Thread contract: the softmax task's
 * (run.rs:1237), as b200rwkv_sample_topk. */
int32_t b200rwkv_sample_probs(b200rwkv_engine*, int32_t nrows, const int32_t* slots, const int32_t* penalty_offset,
                              const uint32_t* penalty_token, const float* penalty_value, const uint32_t* allow_bits,
                              const int32_t* bias_offset, const uint32_t* bias_token, const float* bias_value, float* probs_out);

/* Pinned host memory for logits / state buffers (full-rate DMA); optional. */
int32_t b200rwkv_host_alloc(size_t bytes, void** out);
void b200rwkv_host_free(void* p);

/* Measurement hook used by bench.py for the kernel-resident number: runs `warmup + steps`
 * decode steps (one token per listed slot per step) with token ids staged in HBM beforehand,
 * no host<->device traffic inside the timed region; returns CUDA-event milliseconds for the
 * `steps` timed steps and the number of kernel launches in that region.
 * The steps are real: they compute bit for bit what b200rwkv_infer computes for the same tokens fed one LAST step at a
 * time, so every listed slot's state advances by warmup + steps tokens and its kept row becomes the last step's row.
 * Refused before any CUDA call, with nothing changed: nslot outside [1, max_batch], a duplicate slot, a token id >=
 * num_vocab, steps < 1 or warmup < 0 are B200RWKV_ERR_INVALID; a slot out of range B200RWKV_ERR_STATE.  The two profiling
 * calls below make the same slot, token and nslot checks. */
int32_t b200rwkv_bench_decode(b200rwkv_engine*, int32_t nslot, const int32_t* slot,
                              const uint32_t* tokens /* [(warmup+steps) * nslot] */, int32_t warmup,
                              int32_t steps, int32_t flush_l2, float* ms_out, int64_t* launches_out,
                              float* step_ms_out /* optional [steps]: CUDA-event time of every timed step */);

/* Per-kernel-class device time of ONE un-graphed decode step, CUDA events around every launch
 * on the engine's stream.  classes: 0 = projection GEMMs, 1 = WKV, 2 = LN/mix/embed, 3 = other.
 * ms[4], launches[4], and the algorithmic weight bytes streamed by the step's GEMM launches.
 * The step is real and fully serialised (no programmatic dependent launch): every listed slot's state advances by its token,
 * bit for bit as a b200rwkv_infer step of the same tokens, and the slots are left without a kept row (as after a NONE entry). */
int32_t b200rwkv_profile_step(b200rwkv_engine*, int32_t nslot, const int32_t* slot,
                              const uint32_t* tokens, float ms[4], int32_t launches[4],
                              int64_t* gemm_weight_bytes);

/* In-situ per-launch windows of ONE graph-replayed decode step (globaltimer stamps written by the kernels themselves):
 * window = [griddepcontrol.wait released, last CTA exit]; consecutive windows cannot overlap, so class sums are <= the step.
 * types[i]: 0 LN / mix, 2 WKV, 6 fused RWKV-6 front half, 1000000 + weight MiB for a projection launch; bytes[i]: algorithmic
 * weight bytes of a projection launch (else 0); start_us / end_us relative to the first stamp of the step, averaged over
 * `reps` replays; step_us = last exit - first entry.  bench.py's `roofline` comes from here.
 * The replays are real steps: every listed slot's state advances reps + 1 times by the same token (a warm-up replay, then
 * `reps`), bit for bit as reps + 1 b200rwkv_infer steps of those tokens, and the slots are left without a kept row. */
int32_t b200rwkv_profile_insitu(b200rwkv_engine*, int32_t nslot, const int32_t* slot, const uint32_t* tokens, int32_t reps,
                                int32_t cap, int32_t* n_out, int32_t* types, double* start_us, double* end_us, int64_t* bytes,
                                double* step_us);

/* Operator-level entry (parity tests): the load-time quantiser on a caller-supplied row-major f16 matrix [N, K] (K % 128 == 0),
 * returned in plain order: codes [N, K] (one byte per element: Int8 code, NF4 level index 0..15, FP8 E4M3 code, or Int4 code
 * 0..15), p0 [N, K/block] (Int8, Int4: block minimum, NF4: block absmax), p1 [N, K/block] (Int8: the scale f16((max - min) / 255),
 * Int4: the scale f16((max - min) / 15); NF4, FP8: unused, may be NULL).  p0 / p1 are f16 bit patterns.  block = 128 (Int8,
 * Int4) or 64 (NF4).  FP8: p0 receives the N f32 row scales instead (4 bytes each, 4N bytes in all). */
int32_t b200rwkv_op_quantize(int32_t device, int32_t quant_type, int32_t N, int32_t K, const uint16_t* w_f16, uint8_t* codes,
                             uint16_t* p0, uint16_t* p1);

/* Operator-level entry (parity tests): one WKV launch of a forward step -- recurrence + per-head GroupNorm (eps 64e-5)
 * (+ v7 bonus) * gate, with the step's metadata, grid, kernel choice and launch attributes -- on caller-supplied head vectors
 * and a state pool, no model.  H heads of size 64 (C = H*64 channels), a pool of S slots, and `nslot` step entries: entry i
 * feeds count[i] >= 1 tokens to pool slot slot[i] (distinct slots); its tokens are rows sum(count[0..i]) .. of every per-token
 * array, T = sum(count) <= 128.
 *   r, k, v, g: [T][C] f32 (g is the gate the output is multiplied by); w: decay in (0, 1), [T][C] (v5: static [C]; v6 with
 *   the fold: unused); u: v5 / v6 time_first [C]; lnx_w / lnx_b [C]: ln_x weight and bias.
 *   v7: a [T][C], k_k / k_a / r_k [C] (kk = normalize_head(k * k_k), k <- k * (1 + (a - 1) * k_a), bonus = sum_head(r k r_k));
 *   v_first [T][C] in/out: layer0 != 0 writes v into it, later layers mix v <- v + (v_first - v) * nu with nu [T][C].
 *   v6 decay fold (what the engine runs when the decay LoRA rank Dd <= 128, Dd % 8 == 0): pass d1 [T][Dd] f32 (the LoRA's
 *   tanh stage, rounded to the f16 operand on the device, or hi + lo with precision 1), time_decay_w2 [C][Dd] f16 bits as
 *   stored in the model, decay_bias [C] (time_decay) and Dd; then w = exp(-exp(decay_bias + time_decay_w2 . d1)).
 *   state: in/out [S][H][64][64] in the device orientation M[value][key] (v5/v6: the transpose of S[key][value]).
 *   precision 0: out holds f16 outputs; 1 (T <= 16): split outputs, hi at row t and lo at row t + 16.
 *   out: [rows][C] f16 bits, de-tiled, rows = 16 x token tiles of the step (16 / 32 / 64 / 128 by T; 32 with precision 1).
 *   The caller's contents are uploaded first: cells the kernel does not write come back unchanged.
 *   Snapshots (nsnap 0 / NULL arrays: none), as a step of b200rwkv_infer_snapshots takes them: snap_tok [nsnap] distinct step
 *   token rows in [0, T); snap_rec [nsnap][snap_ld] f32 in/out, uploaded first, where record k receives the state after token
 *   snap_tok[k] at snap_rec[k] + snap_off + h * 4096 (the layout of one slot of `state`); snap_ld >= snap_off + H * 4096,
 *   and snap_off and snap_ld are multiples of 4 (the kernels store records as 16-byte vectors). */
typedef struct {
    int32_t version, H, S, nslot;
    const int32_t *slot, *count;
    int32_t precision;
    const float *r, *k, *v, *g, *w, *u;
    const float *lnx_w, *lnx_b;
    const float *a, *k_k, *k_a, *r_k, *nu;
    int32_t layer0;
    float* v_first;
    const float* d1;
    const uint16_t* time_decay_w2;
    const float* decay_bias;
    int32_t Dd;
    float* state;
    uint16_t* out;
    int32_t nsnap;
    const int32_t* snap_tok;
    float* snap_rec;
    int64_t snap_ld, snap_off;
} b200rwkv_wkv_args;
int32_t b200rwkv_op_wkv(int32_t device, const b200rwkv_wkv_args* args);

/* Operator-level entry (parity tests): one LN stage of a forward step -- with the step's metadata, kernel choice, cluster
 * and launch attributes and token-row layout -- on caller-supplied rows and a pool of S slots, no model.  Entries as in
 * b200rwkv_op_wkv (nslot entries, count[i] >= 1 tokens for distinct pool slot slot[i], T = sum(count) <= 128); C is a
 * multiple of 64, <= 8192.  `launches` (1..16) runs the stage back to back on one stream; per-token arrays carry a
 * leading [launches] dimension, the pool arrays (shift_state, commit_dst) and the front half's barrier counters are shared.
 *   stage 0 embed + LN0:  x_out[t] = LN0(f32(emb[tokens[t]])), emb [V][C] f16 bits, tokens [T] (< V), ln_w / ln_b = ln0.
 *   stage 1 LN / mix (LN1, LN2):  a = x_in + g (.) sum_p parts[p]  (g: gate block c / (C / n_gate) of column c, 1 without
 *     gates), x_out = a, xx = LN(a) (eps 1e-5), prev = shift_state[slot] for an entry's first token, else the LN of the
 *     previous token's a; sx = prev - xx; mix_j = xx + sx mu_j (n_mix 1..6).  commit_dst[slot] <- commit_src[last token of
 *     the entry] (both or neither); hidden (may be NULL) <- a through a device-resident table cell, as the engine records
 *     layers; x_out NULL: in place (x_out is x_in, n_parts = 0), x_in then comes back as the device left it.
 *   stage 2 RWKV-6 front half (T <= 16, Dm 32 or 64, C % 128 == 0, C <= 4096): stage 1 with n_mix = 1 (mu = time_mix_x),
 *     then lora_j = tanh(W1_j mix_0) and out_j = xx + sx (mu5_j + W2_j lora_j), j < 5; W1 [5 Dm][C], W2 [5][C][Dm] f16 bits.
 *   stage 3 ln_out:  a as in stage 1, head row option-row(t) = LN(a) for tokens that produce logits (option per entry:
 *     OPTION_LAST / FULL / NONE), hidden (may be NULL) <- a, the commit as in stage 1.
 *   n_parts, n_gate 0..8: parts [n_parts][T][C], gates [n_gate][T][C / n_gate] (C / n_gate a multiple of 4).
 *   Outputs: x_out, xx_out, sx_out, hidden [T][C] f32; mix_out [n_mix][rows][C], lora_out [5][rows][Dm], out5 [5][rows][C],
 *   head_out [rows][C] f16 bits, de-tiled; rows = 16 x token tiles (16 / 32 / 64 / 128 by T, for head_out by the logits
 *   rows) or 32 with precision 1 (T <= 16), where hi sits at row t and lo at row t + 16.  The caller's contents are uploaded
 *   first: cells the kernel does not write come back unchanged.  kernel_out (may be NULL) receives {kernel, variant, split}:
 *   kernel 0 embed_ln0, 1 ln_mix, 2 ln_mix_cluster, 3 pre6 (variant Dm / 16), 4 ln_out; variant of the other kernels =
 *   float4 per thread (1 / 2 / 4 / 8; always 1 in ln_mix_cluster).
 *   Snapshots (nsnap 0 / NULL arrays: none; stages 1-3, launches 1), as a step of b200rwkv_infer_snapshots takes them:
 *   snap_tok [nsnap] distinct step token rows in [0, T); snap_rec [nsnap][snap_ld] f32 in/out, uploaded first, snap_ld >=
 *   snap_off + C, snap_off and snap_ld multiples of 4 (the kernels store records as 16-byte vectors).  A stage that commits
 *   (commit_src / commit_dst given; ln_out requires it) copies commit_src row snap_tok[k] to snap_rec[k] + snap_off; without
 *   a commit the records are left alone.  ln_out also writes LN(a) of every snapshot token that has no head row, the k-th
 *   such token of snap_tok at row k, into snap_head_out [rows_x][C] f16 bits (required with ln_out snapshots), de-tiled:
 *   rows_x = 32 with precision 1 (hi at row k, lo at row k + 16), else 16 x mt(X) for X such tokens (mt: 1, 2, 4, 8 token
 *   tiles for X <= 16 / 32 / 64 / 128; when X = 0 it may have no rows and is not read). */
typedef struct {
    int32_t stage, C, S, nslot;
    const int32_t *slot, *count;
    const int32_t* option;
    int32_t precision, launches;
    float* x_in;
    int32_t n_parts, n_gate;
    const float *parts, *gates;
    const float *ln_w, *ln_b;
    const float* shift_state;
    int32_t n_mix;
    const float* mu;
    const float* commit_src;
    float* commit_dst;
    float* hidden;
    float *x_out, *xx_out, *sx_out;
    uint16_t* mix_out;
    int32_t Dm;
    const uint16_t *W1, *W2;
    const float* mu5;
    uint16_t *lora_out, *out5;
    const uint16_t* emb;
    int32_t V;
    const uint32_t* tokens;
    uint16_t* head_out;
    int32_t* kernel_out;
    int32_t nsnap;
    const int32_t* snap_tok;
    float* snap_rec;
    int64_t snap_ld, snap_off;
    uint16_t* snap_head_out;
    /* 1: the step runs as a batch-invariant engine runs it (b200rwkv_options.batch_invariant); stages 1 and 2 then take T
     * up to 128 and, above 16 tokens, launch kernel 5 (ln_mix_cluster WIDE, variant 1) / the LN launch plus kernel 6 (pre6
     * WIDE, variant Dm / 16) when C fits the cluster kernels.  0: as before.  Other values are B200RWKV_ERR_INVALID. */
    int32_t batch_invariant;
} b200rwkv_ln_args;
int32_t b200rwkv_op_ln(int32_t device, const b200rwkv_ln_args* args);

/* Operator-level entry (parity tests): one projection launch -- the engine's planner (stream-K cuts, forced grids, Int8 / NF4 /
 * FP8 / Int4 quantisation at load; quant_type B200RWKV_QUANT_*, SF4 refused) and its projection kernels -- over caller-supplied matrices, no model.  Segment i computes
 * act(x W^T + bias) with W [N, K] (row-major f16 bits) and x [launches][T][K] f32, rounded to the f16 operand on the device
 * (precision 0) or split into an f16 hi + lo pair (precision 1: T <= 16, f16 weights).  act: 0 none, 1 tanh, 2 sigmoid,
 * 3 silu, 4 relu^2, 5 exp(-exp), 6 v7 decay.  out_mode: 0 f32 rows; 1 f16 (the operand layout of a following projection,
 * `grp` columns per destination matrix, 0 = one matrix); 2 f16 ddlerp  lerp_xx + lerp_sx * (lerp_mu + y)  with lerp_xx /
 * lerp_sx [launches][T][N] and lerp_mu [N].  out: [launches][rows][ldo], rows = 16 x token tiles (16 / 32 / 64 / 128 by T;
 * 32 with precision 1, where f16 outputs hold the hi halves in rows 0-15 and the lo halves in rows 16-31), f32 or f16 bits,
 * de-tiled.  The caller's contents are uploaded first: cells the kernel does not write come back unchanged.
 * grid 0 = the production plan, > 0 = forced; the plan runs `launches` times back to back on one stream, launch l on input
 * slice l into output slice l.  plan_out (may be NULL): grid launched, stage blocks, tiles, most CTAs contributing to one tile. */
typedef struct {
    int32_t N, K;
    const uint16_t* w;
    const float* x;
    const float* bias;             /* [N] or NULL */
    int32_t act, out_mode, grp;
    const float *lerp_xx, *lerp_sx, *lerp_mu;
    int32_t ldo;                   /* >= N */
    void* out;
} b200rwkv_gemm_seg;
int32_t b200rwkv_op_gemm(int32_t device, int32_t T, int32_t precision, int32_t quant_type, int32_t grid, int32_t launches,
                         int32_t nseg, const b200rwkv_gemm_seg* seg, int32_t* plan_out);

/* Operator-level entry (parity tests): one W' launch of an adapter plan, as b200rwkv_op_gemm runs one segment (precision 0,
 * one launch) with n (1..8) 128-wide adapter tail k blocks after the segment's own: out = act(x W^T + u e^T + bias) with
 * e [N][128 n] f16 the tail blocks' contents (the engine's f16(alpha B) columns) and u [T][128 n] f16 the operand's tail
 * (what the adapter shrink writes).  quant_type B200RWKV_QUANT_*: NONE is the f16 W' plan; INT8 / NF4 / FP8 / INT4 quantise W
 * as b200rwkv_op_gemm does and keep the tail blocks f16 (FP8's row scales apply to x W^T only).  The tail blocks are built by
 * the engine's own W' planner. */
int32_t b200rwkv_op_gemm_tail(int32_t device, int32_t T, int32_t quant_type, int32_t grid, int32_t n, const b200rwkv_gemm_seg* seg,
                              const uint16_t* tail_e, const uint16_t* tail_u, int32_t* plan_out);

/* Operator-level entry (parity tests): the kept-row gather that ends a step -- the step's metadata and the launch rank 0 of a
 * `world`-rank engine makes after it -- on caller-supplied vocabulary shards and kept rows, no model.  Entries as in
 * b200rwkv_op_ln's ln_out stage (nslot entries, count[i] >= 1 tokens for distinct pool slot slot[i], T = sum(count) <= 128,
 * option[i] OPTION_LAST / FULL / NONE), which give the step R logits rows in entry order.
 *   shards: [world][R][Vl] f32, rank q's logits rows of vocabulary ids [q Vl, (q + 1) Vl); each goes to the device in its own
 *     allocation, as every rank's logits block is.  May be NULL when R = 0.
 *   keep: [S][world * Vl] f32, updated in place.  A slot whose entry has a row for its last token gets that row, gathered from
 *     every shard in rank order; every other slot's row comes back unchanged.
 * world 1..8, Vl >= 1, world * Vl <= 4194304. */
typedef struct {
    int32_t S, nslot;
    const int32_t *slot, *count, *option;
    int32_t world, Vl;
    const float* shards;
    float* keep;
} b200rwkv_keep_args;
int32_t b200rwkv_op_keep(int32_t device, const b200rwkv_keep_args* args);

/* Operator-level entry (parity tests): one of the kernels that prepare weights at load, on caller buffers, with the launch
 * shape the model build gives it.  f16 arrays are bit patterns; only the members of the chosen kind are read.
 *   B200RWKV_WEIGHT_LORA: w [out][in] in / out <- f16(f32(w) + alpha * acc), acc the f32 sum over j < r, in order, of
 *     lora_b[o][j] * lora_a[i][j]: one LoRA pair as b200rwkv_create_ex blends it (lora_b = `<name>.lora.1` [out, r],
 *     lora_a = `<name>.lora.0` [in, r]; r 1..4096).
 *   B200RWKV_WEIGHT_F32: dst[i] = f32(src[i]) * scale + bias, i < n: the model's per-channel vectors.
 *   B200RWKV_WEIGHT_DECAY: dst[i] = expf(-expf(f32(src[i]))), i < n: the RWKV-5 static decay.
 *   B200RWKV_WEIGHT_REPACK: rows [n0, n0 + N) and columns [k0, k0 + K) of src [rows][ld] into the projection kernels' weight
 *     blocks: blocks [ceil(N / 128)][ceil(K / 128)] of [k8 16][row group 16][row 8][8 halves] f16, block (tile, kb) holding
 *     rows tile * 128 + 8 * group + row and columns kb * 128 + 8 * k8 + e of the sub-matrix, zero outside it.
 * n 1..2^30. */
#define B200RWKV_WEIGHT_LORA 0
#define B200RWKV_WEIGHT_F32 1
#define B200RWKV_WEIGHT_DECAY 2
#define B200RWKV_WEIGHT_REPACK 3
typedef struct {
    const uint16_t* src;            /* F32, DECAY: [n]; REPACK: [rows][ld] */
    int64_t n;
    float scale, bias;
    float* dst;
    uint16_t* w;                    /* LORA */
    const uint16_t *lora_b, *lora_a;
    int32_t out, in, r;
    float alpha;
    int32_t rows, ld, n0, k0, N, K; /* REPACK */
    uint16_t* blocks;
} b200rwkv_weight_args;
int32_t b200rwkv_op_weight(int32_t device, int32_t kind, const b200rwkv_weight_args* args);

/* Test entry of the adapter shrink kernel (csrc/adapter.cuh), one launch as a step runs it.  x: T token rows of K f16 operand
 * values ([T][K]; precision 1: [2][T][K], the hi rows then the lo rows), T 1..128 (1..16 with precision 1), K a multiple of 8
 * up to 65536.  lora_a[b]: adapter b + 1's `.lora.0` [K][rank[b]] f16, rank 1..128; ids[t] in 0..n: token t's adapter.
 * tail: the n 128-wide tail blocks of the operand after the launch, [T][n][128] f16 (precision 1: [2][T][n][128]): block
 * ids[t] - 1 of row t holds u = x A^T rounded to the operand format in columns < its rank and zeros above it, every other block
 * zeros.  Arguments are checked before the first CUDA call (B200RWKV_ERR_INVALID). */
int32_t b200rwkv_op_adapter(int32_t device, int32_t T, int32_t K, int32_t precision, int32_t n, const int32_t* rank,
                            const uint16_t* const* lora_a, const int32_t* ids, const uint16_t* x, uint16_t* tail);

/* Kernels launched by this engine's forward steps since creation (graph replays counted by their kernel nodes). */
int32_t b200rwkv_launch_count(b200rwkv_engine*, int64_t* total);

/* The residual stream after the last layer, one [num_emb] f32 row per token -- the hidden state the documented embeddings
 * route returns (reference docs/doc-api/openai.md:376-437).  After b200rwkv_keep_hidden(e, 1) every infer call records the
 * rows of ALL its tokens (entry order, like the token array); without it only the rows of the call's last internal step
 * (<= 128 tokens) are available.  b200rwkv_last_hidden returns the number of rows written (negative status on error). */
int32_t b200rwkv_keep_hidden(b200rwkv_engine*, int32_t enable);
int32_t b200rwkv_last_hidden(b200rwkv_engine*, float* out, size_t cap);

/* The residual stream after any chosen layers: the `layer` parameter of the embeddings route (reference
 * docs/doc-api/openai.md:376-437).  "Layer l" is the f32 residual stream after block l, l in [0, num_layer - 1], before any
 * LayerNorm: x_l = x_{l-1} + att_l + ffn_l, with x_{-1} = ln0(emb[token]).  For l = num_layer - 1 the rows are bit-identical
 * to b200rwkv_last_hidden's.  This is our reading of the documentation's wording; no reference output pins it.
 * b200rwkv_keep_hidden_layers(e, n, layers) makes every following infer call record the rows of ALL its tokens for the n
 * listed layers (entry order, like the token array, across internal steps); n = 0 turns recording off.  At most 8 distinct
 * layers; a layer outside [0, num_layer), a duplicate or n > 8 is B200RWKV_ERR_INVALID, checked before the first CUDA call.
 * Independent of b200rwkv_keep_hidden.  Recording adds no kernel launch and changes no other output.
 * b200rwkv_last_hidden_layer copies layer `layer`'s rows of the most recent infer call ([rows][num_emb] f32) and returns the
 * row count: B200RWKV_ERR_STATE if that call did not record the layer, B200RWKV_ERR_INVALID if `cap` (floats) is too small.
 * In-process tensor parallelism: the residual stream is replicated over the ranks; rank 0 records it. */
int32_t b200rwkv_keep_hidden_layers(b200rwkv_engine*, int32_t n, const int32_t* layers);
int32_t b200rwkv_last_hidden_layer(b200rwkv_engine*, int32_t layer, float* out, size_t cap);

/* One pooled hidden row per entry, reduced on the device: what the embeddings route returns (one [num_emb] vector per input)
 * without storing or copying the rows of every token.  "Layer l" is what it is for b200rwkv_keep_hidden_layers.
 * b200rwkv_keep_hidden_pooled(e, n, layers, mode) makes every following infer / infer_ex call reduce, for each of the n
 * listed layers, the rows of each entry to one f32 [num_emb] row; n = 0 turns it off.  At most 8 distinct layers; a layer
 * outside [0, num_layer), a duplicate, n > 8 or an unknown mode is B200RWKV_ERR_INVALID, checked before the first CUDA call.
 *   B200RWKV_POOL_LAST: the row of the entry's last token in the call, bit-identical to that row of
 *     b200rwkv_last_hidden_layer.
 *   B200RWKV_POOL_MEAN: per channel, the f32 sum of the entry's rows in token order, starting from +0.0 with one
 *     round-to-nearest f32 addition per token, then one round-to-nearest f32 division by the entry's token count.  The
 *     order is fixed: the mean is this function of the rows b200rwkv_last_hidden_layer returns for the same call, bit for
 *     bit, however the call is cut into internal steps (token_chunk_size, other entries sharing the steps).
 * Entries of every option (LAST, FULL, NONE, SCORE) pool alike, and pooling changes no logits, state, kept row or score.  It
 * adds one kernel launch per internal step and no per-token copy.  Independent of b200rwkv_keep_hidden and
 * b200rwkv_keep_hidden_layers: any combination may be on at once and none changes what the others return.
 * b200rwkv_last_hidden_pooled copies layer `layer`'s rows of the most recent infer call, [nslot][num_emb] f32 in entry order,
 * and returns nslot; ntok_out (may be NULL, else nslot ints) receives every entry's token count, so a caller whose input was
 * cut over several infer calls can combine the means itself.  An entry without tokens gives a row of zeros and count 0.
 * B200RWKV_ERR_STATE if that call did not pool the layer, B200RWKV_ERR_INVALID if `cap` (floats) is too small.
 * Tensor parallelism: the residual stream is replicated over the ranks; in process rank 0 pools it, and with one process
 * per GPU every rank's engine can (each reduces its own copy). */
#define B200RWKV_POOL_LAST 0
#define B200RWKV_POOL_MEAN 1
int32_t b200rwkv_keep_hidden_pooled(b200rwkv_engine*, int32_t n, const int32_t* layers, int32_t mode);
int32_t b200rwkv_last_hidden_pooled(b200rwkv_engine*, int32_t layer, float* out, size_t cap, int32_t* ntok_out);

/* The n most likely tokens of every scored row, with their log-probabilities, reduced on the device: an OpenAI-style
 * server's `logprobs` / `top_logprobs` (prompt tokens with `echo`, and generated tokens fed back as SCORE entries) without
 * copying logits rows to the host.  b200rwkv_score_top(e, n) makes every following infer_ex / infer_snapshots call also
 * reduce each scored row -- the row score_out[j] comes from, the slot's kept row for j = 0 included -- to its n best
 * entries; n = 0 (the default) turns it off.
 *   - Order: logit descending, then id ascending (b200rwkv_sample_topk's order on an unadjusted row), NaN entries left out.
 *   - logprob = (x_id - m) - logf(S) with the m and S of the row's score, so the target's entry, if listed, is bit-identical
 *     to score_out[j], and ids[j][0] == argmax_out[j] whenever the row has a finite maximum.
 *   - Special values follow score_out: a row with a NaN gives NaN logprobs (its ids are still ranked over the non-NaN
 *     entries); -inf entries come after the finite ones by ascending id; slots past the row's non-NaN entries, and every
 *     slot of a token with no row, are UINT32_MAX / NaN.
 *   - Two kernel launches after each score launch while n > 0; nothing else changes, and n = 0 launches exactly what an
 *     engine that never set it launches.  The lists reach the host with the scores, in the call's one copy.
 * n outside [0, 128] is B200RWKV_ERR_INVALID; n > 0 on a tensor-parallel engine or with num_vocab > 65536 is
 * B200RWKV_ERR_UNSUPPORTED, all before any CUDA call.
 * b200rwkv_last_score_top copies the most recent infer call's lists, ids_out and logprobs_out [sum of ntok over SCORE
 * entries][n] in score_out's order (`cap` entries each), and returns that row count: B200RWKV_ERR_STATE if that call ran
 * with the setting off, B200RWKV_ERR_INVALID if `cap` is too small or only one output is NULL.  With both NULL it copies
 * nothing and returns the row count. */
int32_t b200rwkv_score_top(b200rwkv_engine*, int32_t top_n);
int32_t b200rwkv_last_score_top(b200rwkv_engine*, uint32_t* ids_out, float* logprobs_out, size_t cap);

/* Test aid: copy a named internal activation buffer of the last layer of the most recent step to the host as f32
 * row-major, one row per token of that step; returns the column count (negative status on error).  Not on the product
 * path.  f32 buffers: x_a, x_b, xx1, sx1, xx2, r, k, v, g, w, a, nu, v_first (RWKV-7: the value rows layer 0 wrote),
 * rr, part_att and part_ffn (split-K slices summed in slice order), hidden.  f16 operands: a_x0..a_x5,
 * a_lora<i>_<m>, a_out, a_kk, and a_head, whose first rows are the step's output rows.  An f16 operand name with the
 * suffix "_lo" reads the lo halves of split (hi + lo) operands; the plain name reads the hi halves.  "_lo" is refused
 * with B200RWKV_ERR_STATE when the most recent step did not run split operands.  On an engine with unblended adapters,
 * the suffix "_tail" on a_x0..a_x5, a_out, a_kk or a_head reads the operand's n_adapters x 128 adapter tail columns (the
 * shrink's u = x A^T of each row in its adapter's block, zeros elsewhere), which start at the operand's own columns
 * rounded up to whole 128-column blocks; "_tail_lo" reads their lo halves under the "_lo" rule.  "_tail" is refused with
 * B200RWKV_ERR_STATE on an engine without adapters. */
int32_t b200rwkv_debug_read(b200rwkv_engine*, const char* name, float* out, size_t cap);

/* Test aid, not on the product path: the weight fills the engine runs for one model tensor (at creation, and again on a weight
 * update or a head format change), read back from the device.  b200rwkv_debug_fills returns how many fills read tensor
 * `name` (0: none).  b200rwkv_debug_fill describes fill i in *info and, unless out is NULL, copies its destination to out
 * (info->bytes bytes), untiled on the host, padding included.  R = tiles * 128 rows, Kp = kb * 128 columns:
 *   SEG, qtype NONE: f16 [R][Kp], the rows [n0, n0 + N) and columns [k0, k0 + K) of the matrix (slice `off` of a 3-D tensor,
 *     row stride ld), zero elsewhere.
 *   SEG, quantised: codes u8 [R][Kp] (one code per byte), then Int8 / Int4: min f16 [R][kb] and scale f16 [R][kb]; NF4: absmax
 *     f16 [R][2 kb]; FP8: scale f32 [R] -- b200rwkv_op_quantize's layout over the padded extent.
 *   SEG with ad_tail > 0 (a W' plan): then the adapter tail blocks, f16 [R][ad_tail * 128].
 *   VEC: f32 [count] = f32(x) * scale + bias of elements [off, off + count).  DECAY: f32 [count] = exp(-exp(x)).  RAW: f16 [count].
 *   FOLD: the k-major time_decay_w2 copy as stored, f16 [N heads][K][64] of rows n0 ...  INIT: f32 [head_size + 2][num_emb],
 *     State::init rows of layer n0.
 * plan: the projection plan a SEG fill writes (base, W' of an adapter plan, or the quantised head of b200rwkv_head_format).
 * A NULL engine or name, an unknown name, i out of range or cap < info->bytes is B200RWKV_ERR_INVALID before any CUDA call,
 * and nothing is written to out. */
#define B200RWKV_FILL_SEG 0
#define B200RWKV_FILL_VEC 1
#define B200RWKV_FILL_DECAY 2
#define B200RWKV_FILL_FOLD 3
#define B200RWKV_FILL_RAW 4
#define B200RWKV_FILL_INIT 5
#define B200RWKV_PLAN_BASE 0
#define B200RWKV_PLAN_ADAPTER 1
#define B200RWKV_PLAN_HEAD 2
typedef struct {
    int32_t kind, qtype, plan;
    int32_t n0, N, k0, K, ld;
    int64_t off;
    int32_t tiles, kb, ad_tail;
    int64_t count;
    float scale, bias;
    uint64_t bytes;
} b200rwkv_fill_info;
int32_t b200rwkv_debug_fills(b200rwkv_engine*, const char* name);
int32_t b200rwkv_debug_fill(b200rwkv_engine*, const char* name, int32_t i, b200rwkv_fill_info* info, void* out, size_t cap);

/* Profiling aid: raw stamp rows of the most recent b200rwkv_profile_insitu replay, one row of 512 uint64 per launch
 * (out = [launches][512]): globaltimer stamps of CTA 0 in [0..7] (entry, past griddepcontrol.wait, phase marks, exit), then
 * {SM id, last MMA issued, exit} of every projection CTA (or {entry, released, phase 1 done} of every CTA of the fused RWKV-6
 * front-half kernel); types[i] = 0 LN, 2 WKV, 6 front half, 1000000 + weight MiB for a projection launch. */
int32_t b200rwkv_debug_trace(b200rwkv_engine*, uint64_t* out, size_t cap, int32_t* types, int32_t* nphase);

/* Profiling aid: one projection launch class timed in isolation over all layers, as a 16-token step runs it.  which: 0.. =
 * the launches between LN1 and WKV of a step of more than 16 tokens (the RWKV-6 ddlerp LoRA launches first), 10 = output
 * projection, 20.. = channel-mix launches, 30 = head; an index with no such launch is B200RWKV_ERR_INVALID. */
int32_t b200rwkv_debug_gemm_time(b200rwkv_engine*, int32_t which, int32_t reps, float* ms_out, int64_t* bytes_out,
                                 uint64_t* trace_out);

const char* b200rwkv_last_error(b200rwkv_engine*);

#ifdef __cplusplus
}
#endif
#endif /* B200RWKV_H */
