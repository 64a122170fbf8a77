"""ctypes binding of include/b200rwkv.h (the C-ABI shared library is the product; this file is
only the Python-side loader used by tests/ and bench.py).

The library is loaded from the package directory (built in-tree by ai00_server_b200.build);
loading fails loudly if it is missing — there is no CPU or eager fallback for any entry point.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200rwkv.so")

OK = 0
ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_STATE = -1, -2, -3, -4
OPTION_LAST, OPTION_FULL, OPTION_NONE = 0, 1, 2
OPTION_SCORE = 3                # b200rwkv_infer_ex only: per-token log-probabilities and argmax ids, no logits rows
POOL_LAST, POOL_MEAN = 0, 1      # b200rwkv_keep_hidden_pooled: the entry's last row / the f32 mean of its rows
TP_HANDLE_BYTES = 128


class Info(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "version", "num_layer", "num_emb", "num_hidden", "num_vocab", "num_head", "head_size",
        "time_mix_adapter", "time_decay_adapter")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


MAX_LORA = 4


class Options(C.Structure):
    """b200rwkv_options (include/b200rwkv.h)."""
    _fields_ = [("struct_bytes", C.c_uint32), ("max_batch", C.c_int32), ("token_chunk_size", C.c_int32), ("precision", C.c_int32),
                ("num_devices", C.c_int32), ("devices", C.c_int32 * 8), ("num_lora", C.c_int32),
                ("lora_st", C.c_void_p * MAX_LORA), ("lora_len", C.c_size_t * MAX_LORA), ("lora_alpha", C.c_float * MAX_LORA),
                ("quant_layers", C.c_int32), ("quant_type", C.c_int32), ("batch_invariant", C.c_int32),
                ("quant_adapters", C.c_int32)]


QUANT_NONE, QUANT_INT8, QUANT_NF4 = 0, 1, 2
QUANT_FP8 = 4             # E4M3 codes + one f32 scale per row (3 is the reference's SF4, not implemented)
QUANT_INT4 = 6            # 4-bit codes + f16 (scale, min) per 128 inputs of a row (5 is unassigned)

# B200RWKV_TARGET_*: the kinds of matrix the places of b200rwkv_create_adapter_places can hold pairs on
TARGET_ATT_R, TARGET_ATT_K, TARGET_ATT_V, TARGET_ATT_G = 1 << 0, 1 << 1, 1 << 2, 1 << 3
TARGET_ATT_O, TARGET_FFN_K, TARGET_FFN_V, TARGET_FFN_R, TARGET_HEAD = 1 << 4, 1 << 5, 1 << 6, 1 << 7, 1 << 8
TARGETS = {"att.receptance": TARGET_ATT_R, "att.key": TARGET_ATT_K, "att.value": TARGET_ATT_V, "att.gate": TARGET_ATT_G,
           "att.output": TARGET_ATT_O, "ffn.key": TARGET_FFN_K, "ffn.value": TARGET_FFN_V, "ffn.receptance": TARGET_FFN_R,
           "head": TARGET_HEAD}


# b200rwkv_weight_src.dtype: tensors handed to b200rwkv_update_weights_device
DTYPE_F16, DTYPE_BF16, DTYPE_F32 = 0, 1, 2


class WeightSrc(C.Structure):
    """b200rwkv_weight_src (include/b200rwkv.h): one model tensor on the engine's device, dense."""
    _fields_ = [("name", C.c_char_p), ("dtype", C.c_int32), ("data", C.c_void_p)]


# b200rwkv_fill_info.kind and .plan: the weight fills b200rwkv_debug_fill reads back
FILL_SEG, FILL_VEC, FILL_DECAY, FILL_FOLD, FILL_RAW, FILL_INIT = range(6)
PLAN_BASE, PLAN_ADAPTER, PLAN_HEAD = range(3)


class FillInfo(C.Structure):
    """b200rwkv_fill_info (include/b200rwkv.h)."""
    _fields_ = [(n, C.c_int32) for n in ("kind", "qtype", "plan", "n0", "N", "k0", "K", "ld")] + [("off", C.c_int64)] + [
                (n, C.c_int32) for n in ("tiles", "kb", "ad_tail")] + [
                ("count", C.c_int64), ("scale", C.c_float), ("bias", C.c_float), ("bytes", C.c_uint64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class GemmSeg(C.Structure):
    """b200rwkv_gemm_seg (include/b200rwkv.h)."""
    _fields_ = [("N", C.c_int32), ("K", C.c_int32), ("w", C.c_void_p), ("x", C.c_void_p), ("bias", C.c_void_p),
                ("act", C.c_int32), ("out_mode", C.c_int32), ("grp", C.c_int32),
                ("lerp_xx", C.c_void_p), ("lerp_sx", C.c_void_p), ("lerp_mu", C.c_void_p), ("ldo", C.c_int32), ("out", C.c_void_p)]


class WkvArgs(C.Structure):
    """b200rwkv_wkv_args (include/b200rwkv.h)."""
    _fields_ = [("version", C.c_int32), ("H", C.c_int32), ("S", C.c_int32), ("nslot", C.c_int32), ("slot", C.c_void_p),
                ("count", C.c_void_p), ("precision", C.c_int32)] + [
                (n, C.c_void_p) for n in ("r", "k", "v", "g", "w", "u", "lnx_w", "lnx_b", "a", "k_k", "k_a", "r_k", "nu")] + [
                ("layer0", C.c_int32), ("v_first", C.c_void_p), ("d1", C.c_void_p), ("time_decay_w2", C.c_void_p),
                ("decay_bias", C.c_void_p), ("Dd", C.c_int32), ("state", C.c_void_p), ("out", C.c_void_p),
                ("nsnap", C.c_int32), ("snap_tok", C.c_void_p), ("snap_rec", C.c_void_p), ("snap_ld", C.c_int64),
                ("snap_off", C.c_int64)]


class LnArgs(C.Structure):
    """b200rwkv_ln_args (include/b200rwkv.h)."""
    _fields_ = [(n, C.c_int32) for n in ("stage", "C", "S", "nslot")] + [
                (n, C.c_void_p) for n in ("slot", "count", "option")] + [
                ("precision", C.c_int32), ("launches", C.c_int32), ("x_in", C.c_void_p), ("n_parts", C.c_int32),
                ("n_gate", C.c_int32)] + [
                (n, C.c_void_p) for n in ("parts", "gates", "ln_w", "ln_b", "shift_state")] + [
                ("n_mix", C.c_int32)] + [
                (n, C.c_void_p) for n in ("mu", "commit_src", "commit_dst", "hidden", "x_out", "xx_out", "sx_out", "mix_out")] + [
                ("Dm", C.c_int32)] + [
                (n, C.c_void_p) for n in ("W1", "W2", "mu5", "lora_out", "out5", "emb")] + [
                ("V", C.c_int32), ("tokens", C.c_void_p), ("head_out", C.c_void_p), ("kernel_out", C.c_void_p),
                ("nsnap", C.c_int32), ("snap_tok", C.c_void_p), ("snap_rec", C.c_void_p), ("snap_ld", C.c_int64),
                ("snap_off", C.c_int64), ("snap_head_out", C.c_void_p), ("batch_invariant", C.c_int32)]


LN_EMBED, LN_MIX, LN_FRONT6, LN_OUT = range(4)                     # b200rwkv_ln_args.stage
K_EMBED, K_LN_MIX, K_LN_MIX_CLUSTER, K_PRE6, K_LN_OUT = range(5)   # kernel_out[0]
K_LN_MIX_CLUSTER_WIDE, K_PRE6_WIDE = 5, 6                          # the batch-invariant mode's steps of > 16 tokens


def op_ln(stage: int, channels: int, slots, counts, launches: int = 1, precision: int = 0, option=None, device: int = 0,
          snap_tok=None, snap_off: int = 0, batch_invariant: bool = False, **arrays):
    """One LN stage of a step (b200rwkv_op_ln), `launches` times back to back.  `arrays` holds the struct's array members by
    name (numpy arrays of the header's element types; absent = NULL); output arrays are updated in place.  Snapshots:
    snap_tok (token rows) with arrays snap_rec [nsnap, snap_ld] f32 and, for ln_out, snap_head_out [rows_x, C] uint16.
    batch_invariant: the step as a batch-invariant engine runs it.  Returns kernel_out: (kernel, variant, split)."""
    slots, counts = np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(counts, np.int32)
    keep = [slots, counts]
    a = LnArgs(stage=stage, C=channels, S=int(arrays.pop("S")), nslot=len(slots), slot=ptr(slots), count=ptr(counts),
               precision=precision, launches=launches, n_parts=int(arrays.pop("n_parts", 0)), n_gate=int(arrays.pop("n_gate", 0)),
               n_mix=int(arrays.pop("n_mix", 0)), Dm=int(arrays.pop("Dm", 0)), V=int(arrays.pop("V", 0)),
               batch_invariant=int(batch_invariant))
    if option is not None:
        option = np.ascontiguousarray(option, np.int32)
        keep.append(option)
        a.option = ptr(option)
    if snap_tok is not None:
        snap_tok = np.ascontiguousarray(snap_tok, np.int32)
        keep.append(snap_tok)
        rec = arrays["snap_rec"]
        assert rec.dtype == np.float32 and rec.ndim == 2 and rec.shape[0] == len(snap_tok)
        a.nsnap, a.snap_tok, a.snap_ld, a.snap_off = len(snap_tok), ptr(snap_tok), rec.shape[1], snap_off
    for name, arr in arrays.items():
        if arr is None:
            continue
        assert isinstance(arr, np.ndarray) and arr.flags.c_contiguous, name
        setattr(a, name, ptr(arr))
    kern = np.zeros(3, np.int32)
    a.kernel_out = ptr(kern)
    check(lib().b200rwkv_op_ln(device, C.byref(a)))
    return tuple(int(v) for v in kern)


ACT_NONE, ACT_TANH, ACT_SIGMOID, ACT_SILU, ACT_RELU2, ACT_EXPNEGEXP, ACT_V7DECAY = range(7)
OUT_F32, OUT_A16, OUT_LERP_A16 = 0, 1, 2


class KeepArgs(C.Structure):
    """b200rwkv_keep_args (include/b200rwkv.h)."""
    _fields_ = [("S", C.c_int32), ("nslot", C.c_int32), ("slot", C.c_void_p), ("count", C.c_void_p), ("option", C.c_void_p),
                ("world", C.c_int32), ("Vl", C.c_int32), ("shards", C.c_void_p), ("keep", C.c_void_p)]


def op_keep(slots, counts, options, shards, keep, device: int = 0):
    """The kept-row gather of a step (b200rwkv_op_keep): shards [world, R, Vl] f32, keep [S, world * Vl] f32 updated in place."""
    sl, cn, op = (np.ascontiguousarray(a, np.int32) for a in (slots, counts, options))
    assert shards.dtype == np.float32 and shards.flags.c_contiguous and shards.ndim == 3
    assert keep.dtype == np.float32 and keep.flags.c_contiguous and keep.shape[1] == shards.shape[0] * shards.shape[2]
    a = KeepArgs(keep.shape[0], len(sl), ptr(sl), ptr(cn), ptr(op), shards.shape[0], shards.shape[2], ptr(shards), ptr(keep))
    check(lib().b200rwkv_op_keep(device, C.byref(a)))


WEIGHT_LORA, WEIGHT_F32, WEIGHT_DECAY, WEIGHT_REPACK = range(4)      # b200rwkv_op_weight kinds


class WeightArgs(C.Structure):
    """b200rwkv_weight_args (include/b200rwkv.h)."""
    _fields_ = [("src", C.c_void_p), ("n", C.c_int64), ("scale", C.c_float), ("bias", C.c_float), ("dst", C.c_void_p),
                ("w", C.c_void_p), ("lora_b", C.c_void_p), ("lora_a", C.c_void_p), ("out", C.c_int32), ("in_", C.c_int32),
                ("r", C.c_int32), ("alpha", C.c_float)] + [
                (n, C.c_int32) for n in ("rows", "ld", "n0", "k0", "N", "K")] + [("blocks", C.c_void_p)]


def op_lora_blend(w16, lora_b, lora_a, alpha: float, device: int = 0):
    """One LoRA pair blended into w16 [out, in] f16 (b200rwkv_op_weight, WEIGHT_LORA): lora_b [out, r], lora_a [in, r] f16.
    Returns the blended f16 matrix."""
    w = np.array(w16, np.float16, copy=True, order="C")
    b, a = np.ascontiguousarray(lora_b, np.float16), np.ascontiguousarray(lora_a, np.float16)
    assert b.shape == (w.shape[0], a.shape[1]) and a.shape[0] == w.shape[1]
    args = WeightArgs(w=ptr(w), lora_b=ptr(b), lora_a=ptr(a), out=w.shape[0], in_=w.shape[1], r=a.shape[1], alpha=alpha)
    check(lib().b200rwkv_op_weight(device, WEIGHT_LORA, C.byref(args)))
    return w


def op_vector(kind: int, src16, scale: float = 1.0, bias: float = 0.0, device: int = 0):
    """f32(src) * scale + bias (WEIGHT_F32) or expf(-expf(f32(src))) (WEIGHT_DECAY) of a flat f16 array, as f32."""
    s = np.ascontiguousarray(src16, np.float16).reshape(-1)
    out = np.empty(s.size, np.float32)
    args = WeightArgs(src=ptr(s), n=s.size, scale=scale, bias=bias, dst=ptr(out))
    check(lib().b200rwkv_op_weight(device, kind, C.byref(args)))
    return out


def op_repack(src16, n0: int, k0: int, N: int, K: int, device: int = 0):
    """Rows [n0, n0 + N) x columns [k0, k0 + K) of src16 [rows, ld] f16 as the projection kernels' weight blocks (WEIGHT_REPACK):
    [ceil(N / 128), ceil(K / 128), 16, 16, 8, 8] f16."""
    s = np.ascontiguousarray(src16, np.float16)
    tiles, kb = -(-N // 128), -(-K // 128)
    out = np.empty((tiles, kb, 16, 16, 8, 8), np.float16)
    args = WeightArgs(src=ptr(s), rows=s.shape[0], ld=s.shape[1], n0=n0, k0=k0, N=N, K=K, blocks=ptr(out))
    check(lib().b200rwkv_op_weight(device, WEIGHT_REPACK, C.byref(args)))
    return out


class InferArgs(C.Structure):
    """b200rwkv_infer_args (include/b200rwkv.h)."""
    _fields_ = [("struct_bytes", C.c_uint32), ("nslot", C.c_int32), ("slot", C.c_void_p), ("ntok", C.c_void_p),
                ("tokens", C.c_void_p), ("option", C.c_void_p), ("logits_out", C.c_void_p), ("logits_cap", C.c_size_t),
                ("rows_out", C.c_void_p), ("score_out", C.c_void_p), ("argmax_out", C.c_void_p)]


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200rwkv error {code}: {msg}")
        self.code = code


# every symbol include/b200rwkv.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("b200rwkv_info_from_st", C.c_int32, [_P, C.c_size_t, C.POINTER(Info)]),
    ("b200rwkv_create", C.c_int32, [_P, C.c_size_t, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    ("b200rwkv_create_ex", C.c_int32, [_P, C.c_size_t, C.POINTER(Options), C.POINTER(_P)]),
    ("b200rwkv_create_adapters", C.c_int32, [_P, C.c_size_t, C.POINTER(Options), C.c_int32, _P, _P, _P, C.POINTER(_P)]),
    ("b200rwkv_bind_adapter", C.c_int32, [_P, C.c_int32, _P, _P]),
    ("b200rwkv_create_adapter_places", C.c_int32, [_P, C.c_size_t, C.POINTER(Options), C.c_int32, C.c_uint32, C.POINTER(_P)]),
    ("b200rwkv_load_adapter", C.c_int32, [_P, C.c_int32, _P, C.c_size_t, C.c_float]),
    ("b200rwkv_unload_adapter", C.c_int32, [_P, C.c_int32]),
    ("b200rwkv_update_weights", C.c_int32, [_P, _P, C.c_size_t]),
    ("b200rwkv_update_weights_device", C.c_int32, [_P, C.c_int32, C.POINTER(WeightSrc)]),
    ("b200rwkv_head_format", C.c_int32, [_P, C.c_int32]),
    ("b200rwkv_create_tp", C.c_int32, [_P, C.c_size_t, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    ("b200rwkv_tp_export", C.c_int32, [_P, _P]),
    ("b200rwkv_tp_connect", C.c_int32, [_P, _P]),
    ("b200rwkv_tp_connect_local", C.c_int32, [C.POINTER(_P), C.c_int32]),
    ("b200rwkv_destroy", None, [_P]),
    ("b200rwkv_get_info", C.c_int32, [_P, C.POINTER(Info)]),
    ("b200rwkv_infer", C.c_int32, [_P, C.c_int32, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    ("b200rwkv_infer_ex", C.c_int32, [_P, C.POINTER(InferArgs)]),
    ("b200rwkv_state_shape", C.c_int32, [_P, C.POINTER(C.c_int64 * 4)]),
    ("b200rwkv_state_init", C.c_int32, [_P, _P]),
    ("b200rwkv_state_load", C.c_int32, [_P, C.c_int32, _P]),
    ("b200rwkv_state_back", C.c_int32, [_P, C.c_int32, _P]),
    ("b200rwkv_state_read", C.c_int32, [_P, C.c_int32, C.POINTER(C.c_uint64)]),
    ("b200rwkv_state_write", C.c_int32, [_P, C.c_int32, C.c_uint64]),
    ("b200rwkv_state_free", C.c_int32, [_P, C.c_uint64]),
    ("b200rwkv_infer_snapshots", C.c_int32, [_P, C.POINTER(InferArgs), C.c_int32, _P, _P, _P]),
    ("b200rwkv_snapshot_back", C.c_int32, [_P, C.c_uint64, _P, _P]),
    ("b200rwkv_snapshot_load", C.c_int32, [_P, _P, _P, C.POINTER(C.c_uint64)]),
    ("b200rwkv_cache_stats", C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("b200rwkv_read_state", C.c_int32, [C.POINTER(Info), _P, C.c_size_t, _P]),
    ("b200rwkv_softmax", C.c_int32, [_P, C.c_int32, _P, _P]),
    ("b200rwkv_sample_topk", C.c_int32, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, _P, _P]),
    ("b200rwkv_sample_probs", C.c_int32, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    ("b200rwkv_host_alloc", C.c_int32, [C.c_size_t, C.POINTER(_P)]),
    ("b200rwkv_host_free", None, [_P]),
    ("b200rwkv_bench_decode", C.c_int32, [_P, C.c_int32, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int64), _P]),
    ("b200rwkv_profile_step", C.c_int32, [_P, C.c_int32, _P, _P, C.POINTER(C.c_float * 4), C.POINTER(C.c_int32 * 4), C.POINTER(C.c_int64)]),
    ("b200rwkv_profile_insitu", C.c_int32, [_P, C.c_int32, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.POINTER(C.c_double)]),
    ("b200rwkv_op_quantize", C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P]),
    ("b200rwkv_op_wkv", C.c_int32, [C.c_int32, C.POINTER(WkvArgs)]),
    ("b200rwkv_op_ln", C.c_int32, [C.c_int32, C.POINTER(LnArgs)]),
    ("b200rwkv_op_gemm", C.c_int32, [C.c_int32] * 7 + [C.POINTER(GemmSeg), C.POINTER(C.c_int32 * 4)]),
    ("b200rwkv_op_gemm_tail", C.c_int32, [C.c_int32] * 5 + [C.POINTER(GemmSeg), _P, _P, C.POINTER(C.c_int32 * 4)]),
    ("b200rwkv_op_keep", C.c_int32, [C.c_int32, C.POINTER(KeepArgs)]),
    ("b200rwkv_op_weight", C.c_int32, [C.c_int32, C.c_int32, C.POINTER(WeightArgs)]),
    ("b200rwkv_op_adapter", C.c_int32, [C.c_int32] * 5 + [_P, _P, _P, _P, _P]),
    ("b200rwkv_launch_count", C.c_int32, [_P, C.POINTER(C.c_int64)]),
    ("b200rwkv_keep_hidden", C.c_int32, [_P, C.c_int32]),
    ("b200rwkv_last_hidden", C.c_int32, [_P, _P, C.c_size_t]),
    ("b200rwkv_keep_hidden_layers", C.c_int32, [_P, C.c_int32, _P]),
    ("b200rwkv_last_hidden_layer", C.c_int32, [_P, C.c_int32, _P, C.c_size_t]),
    ("b200rwkv_keep_hidden_pooled", C.c_int32, [_P, C.c_int32, _P, C.c_int32]),
    ("b200rwkv_last_hidden_pooled", C.c_int32, [_P, C.c_int32, _P, C.c_size_t, _P]),
    ("b200rwkv_score_top", C.c_int32, [_P, C.c_int32]),
    ("b200rwkv_last_score_top", C.c_int32, [_P, _P, _P, C.c_size_t]),
    ("b200rwkv_debug_read", C.c_int32, [_P, C.c_char_p, _P, C.c_size_t]),
    ("b200rwkv_debug_fills", C.c_int32, [_P, C.c_char_p]),
    ("b200rwkv_debug_fill", C.c_int32, [_P, C.c_char_p, C.c_int32, C.POINTER(FillInfo), _P, C.c_size_t]),
    ("b200rwkv_debug_trace", C.c_int32, [_P, _P, C.c_size_t, _P, _P]),
    ("b200rwkv_debug_gemm_time", C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int64), _P]),
    ("b200rwkv_last_error", C.c_char_p, [_P]),
]

_lib = None


def lib() -> C.CDLL:
    """Load libb200rwkv.so; raises if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -m ai00_server_b200.build` "
                              "(there is no CPU fallback for the RWKV engine)")
        l = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(l, name)          # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(code: int, engine=None):
    if code < 0:
        msg = lib().b200rwkv_last_error(engine)
        raise B200Error(code, msg.decode("utf-8", "replace") if msg else "")
    return code


def ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def op_adapter(x, lora_a, ids, precision: int = 0, device: int = 0):
    """One adapter shrink launch (b200rwkv_op_adapter): x [T, K] f16 operand rows (precision 1: [2, T, K], hi then lo),
    lora_a: list of n `.lora.0` matrices [K, r] f16, ids [T] in 0..n.  Returns the tail blocks [T, n, 128] f16
    (precision 1: [2, T, n, 128])."""
    x = np.ascontiguousarray(x, dtype=np.float16)
    T, K = x.shape[-2], x.shape[-1]
    mats = [np.ascontiguousarray(a, dtype=np.float16) for a in lora_a]
    n = len(mats)
    rank = np.array([a.shape[1] for a in mats], np.int32)
    ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in mats])
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    tail = np.zeros(((2,) if precision == 1 else ()) + (T, n, 128), np.float16)
    check(lib().b200rwkv_op_adapter(device, T, K, precision, n, ptr(rank), C.cast(ptrs, C.c_void_p), ptr(ids), ptr(x), ptr(tail)))
    return tail


def info_from_st(st: np.ndarray) -> dict:
    st = np.ascontiguousarray(st, dtype=np.uint8)
    out = Info()
    check(lib().b200rwkv_info_from_st(ptr(st), st.size, C.byref(out)))
    return out.as_dict()


def op_quantize(quant_type: int, w16, device: int = 0):
    """The load-time quantiser on one [N, K] f16 matrix (b200rwkv_op_quantize).  Int8: (codes u8 [N, K], min f16 [N, K/128],
    scale f16 [N, K/128]); NF4: (level indices u8 [N, K], absmax f16 [N, K/64]); FP8: (E4M3 codes u8 [N, K], scale f32 [N]);
    Int4: (codes u8 0..15 [N, K], min f16 [N, K/128], scale f16 [N, K/128])."""
    w16 = np.ascontiguousarray(w16, np.float16)
    N, K = w16.shape
    if quant_type == QUANT_FP8:
        codes = np.empty((N, K), np.uint8)
        scale = np.empty(N, np.float32)
        check(lib().b200rwkv_op_quantize(device, quant_type, N, K, ptr(w16), ptr(codes), ptr(scale), None))
        return codes, scale
    affine = quant_type in (QUANT_INT8, QUANT_INT4)          # (codes, min, scale) per 128-input block
    nb = K // (128 if affine else 64)
    codes = np.empty((N, K), np.uint8)
    p0 = np.empty((N, nb), np.float16)
    p1 = np.empty((N, nb), np.float16)
    check(lib().b200rwkv_op_quantize(device, quant_type, N, K, ptr(w16), ptr(codes), ptr(p0), ptr(p1) if affine else None))
    return (codes, p0, p1) if affine else (codes, p0)


def op_wkv_step(version: int, slots, counts, state, out, r, k, v, g, lnx_w, lnx_b, w=None, u=None, a=None, k_k=None, k_a=None,
                r_k=None, nu=None, layer0: bool = True, v_first=None, d1=None, time_decay_w2=None, decay_bias=None, precision: int = 0,
                snap_tok=None, snap_rec=None, snap_off: int = 0, device: int = 0):
    """One WKV launch of a step (b200rwkv_op_wkv) over a pool of S slots: entry i feeds counts[i] tokens to pool slot slots[i].
    state [S, H, 64, 64] f32 (M[value][key]), out [gemm_rows(T, precision), H*64] uint16 f16 bits and v7's v_first [T, H*64]
    f32 are updated in place.  Per-token arrays are [T, H*64] (or [T, H, 64]) f32, per-channel ones [H*64]; d1 [T, Dd] f32 and
    time_decay_w2 [H*64, Dd] f16 turn on the v6 decay fold.  Snapshots: snap_tok (token rows) and snap_rec [nsnap, snap_ld]
    f32, updated in place: record k receives the state after token snap_tok[k] from column snap_off on."""
    S, H = state.shape[:2]
    assert state.dtype == np.float32 and state.flags.c_contiguous and state.shape[2:] == (64, 64)
    assert out.dtype == np.uint16 and out.flags.c_contiguous and out.shape == (gemm_rows(sum(counts), precision), H * 64)
    assert v_first is None or (v_first.dtype == np.float32 and v_first.flags.c_contiguous)
    f32 = lambda x: None if x is None else np.ascontiguousarray(x, np.float32)
    keep = [np.ascontiguousarray(slots, np.int32), np.ascontiguousarray(counts, np.int32)]
    keep += [f32(x) for x in (r, k, v, g, w, u, lnx_w, lnx_b, a, k_k, k_a, r_k, nu, d1, decay_bias)]
    w2 = None if time_decay_w2 is None else np.ascontiguousarray(time_decay_w2, np.float16)
    p = lambda x: None if x is None else ptr(x)
    sl, cn, r, k, v, g, w, u, lnx_w, lnx_b, a, k_k, k_a, r_k, nu, d1, decay_bias = keep
    args = WkvArgs(version, H, S, len(sl), p(sl), p(cn), precision, p(r), p(k), p(v), p(g), p(w), p(u), p(lnx_w), p(lnx_b), p(a),
                   p(k_k), p(k_a), p(r_k), p(nu), int(layer0), p(v_first), p(d1), p(w2), p(decay_bias),
                   0 if d1 is None else d1.shape[1], ptr(state), ptr(out))
    if snap_tok is not None:
        st_ = np.ascontiguousarray(snap_tok, np.int32)
        keep.append(st_)
        assert snap_rec.dtype == np.float32 and snap_rec.flags.c_contiguous and snap_rec.shape[0] == len(st_)
        args.nsnap, args.snap_tok, args.snap_rec, args.snap_ld, args.snap_off = len(st_), ptr(st_), ptr(snap_rec), snap_rec.shape[1], snap_off
    check(lib().b200rwkv_op_wkv(device, C.byref(args)))


def op_wkv(version: int, r, k, v, w, state, u=None, a=None, k_k=None, k_a=None, r_k=None, g=None, lnx_w=None, lnx_b=None, device: int = 0):
    """One sequence through the WKV kernel (op_wkv_step with one slot; v7 at layer 0).  r, k, v: [T, H, 64]; g None = 1, lnx_w /
    lnx_b None = 1 / 0; state [H, 64, 64] = M[value][key] (updated copy returned).  Returns (out [T, H, 64] f32, state)."""
    r = np.ascontiguousarray(r, np.float32)
    T, H, _ = r.shape
    ones = np.ones(H * 64, np.float32)
    st = np.array(state, np.float32, copy=True, order="C")[None]
    out = np.zeros((gemm_rows(T), H * 64), np.uint16)
    v_first = np.zeros((T, H * 64), np.float32) if version == 7 else None
    op_wkv_step(version, [0], [T], st, out, r, k, v, np.ones((T, H * 64), np.float32) if g is None else g,
                ones if lnx_w is None else lnx_w, ones * 0 if lnx_b is None else lnx_b, w=w, u=u, a=a, k_k=k_k, k_a=k_a, r_k=r_k,
                v_first=v_first, device=device)
    return out[:T].view(np.float16).astype(np.float32).reshape(T, H, 64), st[0]


def gemm_rows(T: int, precision: int = 0) -> int:
    """Token rows of b200rwkv_op_gemm's outputs: 16 x the token tiles of the kernel the engine runs for T tokens."""
    if precision == 1:
        return 32
    return 16 if T <= 16 else 32 if T <= 32 else 64 if T <= 64 else 128


def op_gemm(T: int, segs: list[dict], precision: int = 0, quant_type: int = QUANT_NONE, grid: int = 0, launches: int = 1,
            device: int = 0):
    """One projection launch (b200rwkv_op_gemm).  Each segment is a dict: w [N, K] f16, x [launches, T, K] f32, optional bias
    [N], act, out_mode, grp, xx / sx [launches, T, N] and mu [N] (ddlerp), and out [launches, gemm_rows(T), ldo] (float32 for
    OUT_F32, uint16 f16 bits otherwise), whose contents are uploaded first and overwritten in place where the kernel writes.
    Returns the plan: (grid, stage blocks, tiles, most contributing CTAs of one tile)."""
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    keep, arr = [], (GemmSeg * len(segs))()
    for i, d in enumerate(segs):
        w = np.ascontiguousarray(d["w"], np.float16)
        x, bias, xx, sx, mu = (f32(d.get(k)) for k in ("x", "bias", "xx", "sx", "mu"))
        out = d["out"]
        assert out.flags.c_contiguous and out.dtype == (np.float32 if d.get("out_mode", OUT_F32) == OUT_F32 else np.uint16)
        assert x.shape == (launches, T, w.shape[1]) and out.shape[:2] == (launches, gemm_rows(T, precision))
        keep += [w, x, bias, xx, sx, mu]
        p = lambda a: None if a is None else ptr(a)
        arr[i] = GemmSeg(w.shape[0], w.shape[1], p(w), p(x), p(bias), d.get("act", ACT_NONE), d.get("out_mode", OUT_F32),
                         d.get("grp", 0), p(xx), p(sx), p(mu), out.shape[2], ptr(out))
    plan = (C.c_int32 * 4)()
    check(lib().b200rwkv_op_gemm(device, T, precision, quant_type, grid, launches, len(segs), arr, C.byref(plan)))
    return tuple(plan)


def op_gemm_tail(T: int, seg: dict, e: np.ndarray, u: np.ndarray, quant_type: int = QUANT_NONE, grid: int = 0, device: int = 0):
    """One W' launch of an adapter plan (b200rwkv_op_gemm_tail): `seg` as one op_gemm segment with launches = 1 (x [1, T, K],
    out [1, gemm_rows(T), ldo]), plus n = e.shape[1] / 128 tail blocks with contents e [N, 128 n] f16 and the operand's tail
    u [T, 128 n] f16.  Returns the plan as op_gemm does."""
    w = np.ascontiguousarray(seg["w"], np.float16)
    x = np.ascontiguousarray(seg["x"], np.float32)
    bias = None if seg.get("bias") is None else np.ascontiguousarray(seg["bias"], np.float32)
    out = seg["out"]
    e = np.ascontiguousarray(e, np.float16)
    u = np.ascontiguousarray(u, np.float16)
    n = e.shape[1] // 128
    assert out.flags.c_contiguous and out.dtype == (np.float32 if seg.get("out_mode", OUT_F32) == OUT_F32 else np.uint16)
    assert x.shape == (1, T, w.shape[1]) and out.shape[:2] == (1, gemm_rows(T))
    assert e.shape == (w.shape[0], 128 * n) and u.shape == (T, 128 * n)
    s = GemmSeg(w.shape[0], w.shape[1], ptr(w), ptr(x), None if bias is None else ptr(bias), seg.get("act", ACT_NONE),
                seg.get("out_mode", OUT_F32), seg.get("grp", 0), None, None, None, out.shape[2], ptr(out))
    plan = (C.c_int32 * 4)()
    check(lib().b200rwkv_op_gemm_tail(device, T, quant_type, grid, n, C.byref(s), ptr(e), ptr(u), C.byref(plan)))
    return tuple(plan)
