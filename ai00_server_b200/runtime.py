"""Host-side mirror of the web-rwkv interface that crates/ai00-core consumes, over the C ABI.

The reference's host code is Rust (crates/ai00-core/src/run.rs, lib.rs) and no Rust toolchain
exists in this image, so the shim that would live in ai00-core is specified in INTEGRATION.md
and mirrored here 1:1 in Python for the parity tests and bench.py: same names, argument
meaning and error behaviour as the trait objects the reference holds:

  RnnOption / RnnInputBatch / RnnInput / RnnOutputBatch   run.rs:25, 1121-1136, 1146
  Runtime.infer(input) -> (input, output)                   run.rs:1143
  State.{init, load, back, read, write}                     run.rs:477, 1099-1107
  softmax(list of [V] tensors)                              run.rs:1179
  Loader.info                                               lib.rs:587
  ModelBuilder(...).build() + Bundle(model, max_batch)      lib.rs:484-497

Every method calls straight into libb200rwkv.so; nothing here computes on the CPU.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import enum
from dataclasses import dataclass, field

import numpy as np

from . import capi


class RnnOption(enum.IntEnum):
    Last = capi.OPTION_LAST
    Full = capi.OPTION_FULL


@dataclass
class RnnInputBatch:
    tokens: list = field(default_factory=list)
    option: RnnOption = RnnOption.Last


@dataclass
class RnnInput:
    batches: list
    token_chunk_size: int

    def num_token(self) -> int:
        return sum(len(b.tokens) for b in self.batches)


@dataclass
class RnnOutputBatch:
    """`RnnOutputBatch(TensorCpu<f32>)`: [rows, V]; empty when the slot produced nothing."""
    data: np.ndarray

    def is_empty(self) -> bool:
        return self.data.shape[0] == 0


class Loader:
    @staticmethod
    def info(st: np.ndarray) -> dict:
        return capi.info_from_st(st)


def read_state(info: dict, st: np.ndarray) -> np.ndarray:
    """`vN::read_state(&context, &info, reader)` (lib.rs:378-389): `.state` file / state-tuned model -> state tensor."""
    st = np.ascontiguousarray(st, dtype=np.uint8)
    ci = capi.Info(**{k: int(v) for k, v in info.items()})
    out = np.empty((info["num_layer"], info["head_size"] + 2, info["num_emb"]), np.float32)
    capi.check(capi.lib().b200rwkv_read_state(C.byref(ci), capi.ptr(st), st.size, capi.ptr(out)))
    return out


def quant_kind(kind, what: str = "quant_type") -> int:
    """A weight format's B200RWKV_QUANT_* value from its name (any case: None, Int8, NF4, SF4, FP8, Int4); an int is passed
    through for the engine to check."""
    if not isinstance(kind, str):
        return int(kind)
    kinds = {"none": capi.QUANT_NONE, "int8": capi.QUANT_INT8, "nf4": capi.QUANT_NF4, "sf4": 3, "fp8": capi.QUANT_FP8,
             "int4": capi.QUANT_INT4}
    if kind.lower() not in kinds:
        raise capi.B200Error(capi.ERR_INVALID, f"{what} must be None, Int8, NF4, SF4, FP8 or Int4")
    return kinds[kind.lower()]


def _fill_parts(info: dict, raw: np.ndarray, head_size: int, num_emb: int) -> dict:
    """The parts of one b200rwkv_debug_fill read-back (Model.debug_fills)."""
    kind = info["kind"]
    if kind == capi.FILL_VEC or kind == capi.FILL_DECAY:
        return {"v": raw.view(np.float32)}
    if kind == capi.FILL_RAW:
        return {"v": raw.view(np.uint16)}
    if kind == capi.FILL_FOLD:
        return {"v": raw.view(np.uint16).reshape(info["N"], info["K"], 64)}
    if kind == capi.FILL_INIT:
        return {"v": raw.view(np.float32).reshape(head_size + 2, num_emb)}
    R, kb, qt = info["tiles"] * 128, info["kb"], info["qtype"]
    Kp, o, parts = kb * 128, 0, {}

    def take(name, dtype, shape):
        nonlocal o
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        parts[name] = raw[o:o + n].view(dtype).reshape(shape)
        o += n

    if qt == capi.QUANT_NONE:
        take("w", np.uint16, (R, Kp))
    else:
        take("codes", np.uint8, (R, Kp))
        if qt == capi.QUANT_FP8:
            take("scale", np.float32, (R,))
        elif qt == capi.QUANT_NF4:
            take("absmax", np.float16, (R, 2 * kb))
        else:
            take("min", np.float16, (R, kb))
            take("scale", np.float16, (R, kb))
    if info["ad_tail"]:
        take("tail", np.uint16, (R, info["ad_tail"] * 128))
    assert o == raw.size
    return parts


class TensorGpu:
    """Device-side state snapshot handle (`TensorGpu<f32, ReadWrite>` at run.rs:1104-1108)."""

    def __init__(self, model: "Model", snap_id: int):
        self._model, self.id = model, snap_id

    def free(self):
        if self.id:
            capi.check(capi.lib().b200rwkv_state_free(self._model._h, self.id), self._model._h)
            self.id = 0


class State:
    def __init__(self, model: "Model"):
        self._m = model

    def shape(self):
        s = (C.c_int64 * 4)()
        capi.check(capi.lib().b200rwkv_state_shape(self._m._h, C.byref(s)), self._m._h)
        return tuple(s)

    def _numel(self):
        s = self.shape()
        return int(s[0] * s[1] * s[2] * s[3])

    def _np_shape(self):
        c, r, l, _ = self.shape()
        return (int(l), int(r), int(c))        # numpy C-order view of web-rwkv [C, N+2, L, 1]

    def init(self) -> np.ndarray:
        out = np.empty(self._np_shape(), np.float32)
        capi.check(capi.lib().b200rwkv_state_init(self._m._h, capi.ptr(out)), self._m._h)
        return out

    def load(self, tensor: np.ndarray, batch: int) -> None:
        t = np.ascontiguousarray(tensor, dtype=np.float32)
        if t.size != self._numel():
            raise capi.B200Error(capi.ERR_INVALID, "state tensor has the wrong number of elements")
        capi.check(capi.lib().b200rwkv_state_load(self._m._h, batch, capi.ptr(t)), self._m._h)

    def back(self, batch: int) -> np.ndarray:
        out = np.empty(self._np_shape(), np.float32)
        capi.check(capi.lib().b200rwkv_state_back(self._m._h, batch, capi.ptr(out)), self._m._h)
        return out

    def read(self, batch: int) -> TensorGpu:
        sid = C.c_uint64(0)
        capi.check(capi.lib().b200rwkv_state_read(self._m._h, batch, C.byref(sid)), self._m._h)
        return TensorGpu(self._m, sid.value)

    def write(self, tensor: TensorGpu, batch: int) -> None:
        capi.check(capi.lib().b200rwkv_state_write(self._m._h, batch, tensor.id), self._m._h)

    # ---- device-resident cache items (CachedItem {state, output}, run.rs:199-205) ----
    def snapshot_back(self, tensor: TensorGpu, with_logits: bool = False):
        out = np.empty(self._np_shape(), np.float32)
        lg = np.empty(self._m.info["num_vocab"], np.float32) if with_logits else None
        capi.check(capi.lib().b200rwkv_snapshot_back(self._m._h, tensor.id, capi.ptr(out), capi.ptr(lg) if with_logits else None), self._m._h)
        return (out, lg) if with_logits else out

    def snapshot_load(self, tensor: np.ndarray, logits: np.ndarray | None = None) -> TensorGpu:
        t = np.ascontiguousarray(tensor, dtype=np.float32)
        if t.size != self._numel():
            raise capi.B200Error(capi.ERR_INVALID, "state tensor has the wrong number of elements")
        lg = None if logits is None else np.ascontiguousarray(logits, dtype=np.float32)
        sid = C.c_uint64(0)
        capi.check(capi.lib().b200rwkv_snapshot_load(self._m._h, capi.ptr(t), capi.ptr(lg) if lg is not None else None, C.byref(sid)), self._m._h)
        return TensorGpu(self._m, sid.value)

    def cache_stats(self) -> dict:
        n, used, free = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        capi.check(capi.lib().b200rwkv_cache_stats(self._m._h, C.byref(n), C.byref(used), C.byref(free)), self._m._h)
        return {"snapshots": n.value, "bytes_used": used.value, "bytes_free": free.value}


class NucleusSampler:
    """Host back half of the reference's `NucleusSampler` (sampler/nucleus.rs:13-123) over the <= 128 candidates the GPU
    front half returns: same parameters, same penalty state, same arithmetic in f32; `rand` is the uniform draw the
    reference takes from fastrand (nucleus.rs:104), passed in so tests are deterministic."""

    def __init__(self, top_p=0.5, top_k=128, temperature=1.0, presence_penalty=0.3, frequency_penalty=0.3,
                 penalty_decay=0.99654026):
        f = np.float32
        self.top_p, self.top_k, self.temperature = f(top_p), int(top_k), f(temperature)
        self.presence_penalty, self.frequency_penalty, self.penalty_decay = f(presence_penalty), f(frequency_penalty), f(penalty_decay)
        self.penalties: dict[int, np.float32] = {}

    def init(self, model_tokens):                                   # nucleus.rs:50-59
        for index, token in enumerate(reversed(list(model_tokens))):
            pen = self.penalties.pop(int(token), self.presence_penalty)
            pen = np.float32(pen + self.frequency_penalty * np.float32(np.power(self.penalty_decay, np.float32(index))))
            self.penalties[int(token)] = pen

    def sample_candidates(self, ids, probs, rand: float) -> int:   # nucleus.rs:69-123 after the sort / take(top_k)
        f = np.float32
        kept, cum = [], f(0.0)
        for i, x in zip(ids[:self.top_k], probs[:self.top_k]):
            if cum > self.top_p:
                break
            cum = f(cum + x)
            kept.append((int(i), f(np.power(f(x), f(1.0) / self.temperature))))
        total = f(0.0)
        for _, x in kept:
            total = f(total + x)
        token, cum = kept[0][0], f(0.0)
        for i, x in kept:
            cum = f(cum + f(x / total))
            if f(rand) <= cum:
                token = i
                break
        for t in self.penalties:
            self.penalties[t] = f(self.penalties[t] * self.penalty_decay)
        self.penalties[token] = f(self.penalties[token] + self.frequency_penalty) if token in self.penalties else self.presence_penalty
        return token


class Runtime:
    """`Arc<dyn Runtime<Rnn>>`.  `infer` consumes at most `token_chunk_size` tokens of the
    input across slots and returns the remaining input with the per-slot outputs, exactly the
    contract the batching shim loops on (run.rs:1134-1155)."""

    def __init__(self, model: "Model"):
        self._m = model

    def infer(self, inp: RnnInput):
        m = self._m
        budget = max(1, inp.token_chunk_size)
        slots, ntok, opts, toks, takes = [], [], [], [], []
        for b, batch in enumerate(inp.batches):
            if not batch.tokens or budget == 0:
                takes.append(0)
                continue
            take = min(len(batch.tokens), budget)
            budget -= take
            takes.append(take)
            finishes = take == len(batch.tokens)
            slots.append(b)
            ntok.append(take)
            toks.extend(int(t) for t in batch.tokens[:take])
            # Last only yields a row once the slot's tokens are exhausted
            opts.append(int(RnnOption.Full) if batch.option == RnnOption.Full
                        else (int(RnnOption.Last) if finishes else capi.OPTION_NONE))
        rows = m.infer_raw(slots, ntok, toks, opts)
        out = [RnnOutputBatch(np.zeros((0, m.info["num_vocab"]), np.float32)) for _ in inp.batches]
        for s, r in zip(slots, rows):
            out[s] = RnnOutputBatch(r)
        rest = RnnInput([RnnInputBatch(list(b.tokens[t:]), b.option) for b, t in zip(inp.batches, takes)],
                        inp.token_chunk_size)
        return rest, out


class Model:
    """Owns one engine (`ModelBuilder...build_vN()` + `Bundle::new(model, max_batch)` +
    `TokioRuntime::new(bundle)`, lib.rs:484-497)."""

    def __init__(self, st: np.ndarray, max_batch: int = 8, token_chunk_size: int = 128, device: int = 0,
                 precision: int = 0, rank: int = 0, world: int = 1, exact: bool = False, devices=None, lora=None,
                 quant: int = 0, quant_type: int | str = 0, adapters=None, adapter_places: int = 0,
                 adapter_targets=(), batch_invariant: bool = False, quant_adapters: bool = False, quant_head=None):
        """devices: list of CUDA ordinals -> ONE engine object owning all tensor-parallel ranks (b200rwkv_create_ex);
        lora: list of (st_bytes, alpha) blended at load (reference lib.rs:466-485);
        quant / quant_type: the reload request's fields (lib.rs:211-215): the first `quant` layers in "Int8" or "NF4",
        or in "FP8" (E4M3 codes with one scale per row) or "Int4" (4-bit codes with (scale, min) per 128 inputs), this
        project's own formats;
        rank / world: one process per GPU instead (b200rwkv_create_tp + tp.connect);
        adapters: list of (st_bytes, alpha) kept unblended, ids 1..n, chosen per slot with bind_adapter
        (b200rwkv_create_adapters);
        adapter_places / adapter_targets: n empty adapter places, filled and emptied with load_adapter / unload_adapter,
        that hold pairs on the named kinds of matrix ("att.key", ..., "head": the keys of capi.TARGETS)
        (b200rwkv_create_adapter_places);
        batch_invariant: every token's results are the bits a decode step gives it, whatever else shares its calls
        (b200rwkv_options.batch_invariant);
        quant_adapters: adapters and adapter places may pair matrices of the quantised layers
        (b200rwkv_options.quant_adapters);
        quant_head: the vocabulary head's weight format, a quant_type value, set right after creation with head_format()
        (None: the f16 head)."""
        quant_type = quant_kind(quant_type)
        head_kind = None if quant_head is None else quant_kind(quant_head, "quant_head")
        quantised = quant > 0 and quant_type != capi.QUANT_NONE
        if exact:
            precision = 1          # `Bundle::<f32>`: f32-exact activations (split hi + lo f16 operands)
        st = np.ascontiguousarray(st, dtype=np.uint8)
        h = C.c_void_p()
        L = capi.lib()
        if adapters and adapter_places:
            raise capi.B200Error(capi.ERR_INVALID, "adapters and adapter_places are two constructors: pass one")
        if devices is not None or lora or quantised or adapters or adapter_places or batch_invariant or quant_adapters:
            if world != 1:
                raise capi.B200Error(capi.ERR_INVALID, "devices / lora / quant go through b200rwkv_create_ex (in-process ranks)")
            opt = capi.Options()
            opt.struct_bytes = C.sizeof(capi.Options)
            opt.max_batch, opt.token_chunk_size, opt.precision = max_batch, token_chunk_size, precision
            devs = list(devices) if devices is not None else [device]
            opt.num_devices = len(devs)
            for i, d in enumerate(devs):
                opt.devices[i] = int(d)
            self._lora_keep = []
            for i, (img, alpha) in enumerate(lora or []):
                img = np.ascontiguousarray(img, dtype=np.uint8)
                self._lora_keep.append(img)
                opt.lora_st[i], opt.lora_len[i], opt.lora_alpha[i] = img.ctypes.data, img.size, float(alpha)
            opt.num_lora = len(lora or [])
            opt.quant_layers, opt.quant_type = (int(quant), int(quant_type)) if quantised else (0, 0)
            opt.batch_invariant = int(bool(batch_invariant))
            opt.quant_adapters = int(bool(quant_adapters))
            if adapters:
                imgs = [np.ascontiguousarray(img, dtype=np.uint8) for img, _ in adapters]
                n = len(imgs)
                ptrs = (C.c_void_p * n)(*[img.ctypes.data for img in imgs])
                lens = (C.c_size_t * n)(*[img.size for img in imgs])
                alphas = (C.c_float * n)(*[float(a) for _, a in adapters])
                capi.check(L.b200rwkv_create_adapters(capi.ptr(st), st.size, C.byref(opt), n, C.cast(ptrs, C.c_void_p),
                                                      C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p), C.byref(h)))
            elif adapter_places:
                unknown = [t for t in adapter_targets if t not in capi.TARGETS]
                if unknown:
                    raise capi.B200Error(capi.ERR_INVALID, f"unknown adapter targets {unknown}: use keys of capi.TARGETS")
                mask = 0
                for t in adapter_targets:
                    mask |= capi.TARGETS[t]
                capi.check(L.b200rwkv_create_adapter_places(capi.ptr(st), st.size, C.byref(opt), int(adapter_places), mask,
                                                            C.byref(h)))
            else:
                capi.check(L.b200rwkv_create_ex(capi.ptr(st), st.size, C.byref(opt), C.byref(h)))
            self._lora_keep = []
        else:
            capi.check(L.b200rwkv_create_tp(capi.ptr(st), st.size, device, max_batch, token_chunk_size, precision,
                                            rank, world, C.byref(h)))
        self._h = h
        self._top_n = 0                # b200rwkv_score_top setting
        self.max_batch, self.token_chunk_size = max_batch, token_chunk_size
        self.rank, self.world = rank, world
        info = capi.Info()
        capi.check(L.b200rwkv_get_info(self._h, C.byref(info)), self._h)
        self.info = info.as_dict()
        self.runtime = Runtime(self)
        self.state = State(self)
        if head_kind is not None:
            try:
                self.head_format(head_kind)
            except Exception:
                self.close()
                raise

    def close(self):
        if self._h:
            capi.lib().b200rwkv_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- raw call: one b200rwkv_infer ----
    def infer_raw(self, slots, ntok, tokens, options, out: np.ndarray | None = None, keep_on_device: bool = False):
        V = self.info["num_vocab"]          # rank 0 receives the gathered full-vocabulary rows
        n = len(slots)
        total = sum(nt if o == capi.OPTION_FULL else (1 if (o == capi.OPTION_LAST and nt > 0) else 0)
                    for nt, o in zip(ntok, options))
        if keep_on_device:                  # logits_out = NULL: rows stay in HBM for sample_topk
            a_slot, a_ntok = np.asarray(slots, np.int32), np.asarray(ntok, np.int32)
            a_tok, a_opt = np.asarray(tokens, np.uint32), np.asarray(options, np.int32)
            a_rows = np.zeros(max(n, 1), np.int32)
            capi.check(capi.lib().b200rwkv_infer(self._h, n, capi.ptr(a_slot), capi.ptr(a_ntok), capi.ptr(a_tok),
                                                 capi.ptr(a_opt), None, 0, capi.ptr(a_rows)), self._h)
            return [int(r) for r in a_rows[:n]]
        if out is None:
            out = np.empty((max(total, 1), V), np.float32)
        a_slot = np.asarray(slots, np.int32)
        a_ntok = np.asarray(ntok, np.int32)
        a_tok = np.asarray(tokens, np.uint32)
        a_opt = np.asarray(options, np.int32)
        a_rows = np.zeros(max(n, 1), np.int32)
        capi.check(capi.lib().b200rwkv_infer(self._h, n, capi.ptr(a_slot), capi.ptr(a_ntok), capi.ptr(a_tok),
                                             capi.ptr(a_opt), capi.ptr(out), out.size, capi.ptr(a_rows)), self._h)
        res, off = [], 0
        for i in range(n):
            r = int(a_rows[i])
            res.append(out[off:off + r])
            off += r
        return res

    # ---- raw call with scoring: one b200rwkv_infer_ex ----
    def infer_ex(self, slots, ntok, tokens, options, top_n: int | None = None):
        """b200rwkv_infer_ex: `options` may also hold capi.OPTION_SCORE.  Returns (rows, scores): rows per entry as infer_raw
        returns them (0 rows for SCORE entries); scores[i] is (log-probabilities f32 [ntok[i]], argmax ids uint32 [ntok[i]])
        for a SCORE entry, None otherwise.  Token 0 of a SCORE entry is scored from the slot's kept row (NaN if it has none).
        With `top_n` (1..128) the call runs with score_top(top_n) and returns (rows, scores, tops), tops[i] the entry's
        (ids uint32 [ntok[i]][top_n], log-probabilities f32 [ntok[i]][top_n]) for a SCORE entry, None otherwise; the engine's
        own setting is restored afterwards."""
        if top_n is not None:
            with self._score_top_as(top_n):
                rows, scores = self.infer_ex(slots, ntok, tokens, options)
                return rows, scores, self._split_tops(ntok, options, self.last_score_top())
        V = self.info["num_vocab"]
        n = len(slots)
        total = sum(nt if o == capi.OPTION_FULL else (1 if (o == capi.OPTION_LAST and nt > 0) else 0)
                    for nt, o in zip(ntok, options))
        nscore = sum(nt for nt, o in zip(ntok, options) if o == capi.OPTION_SCORE)
        out = np.empty((max(total, 1), V), np.float32)
        score = np.empty(max(nscore, 1), np.float32)
        argmax = np.empty(max(nscore, 1), np.uint32)
        a_slot, a_ntok = np.asarray(slots, np.int32), np.asarray(ntok, np.int32)
        a_tok, a_opt = np.asarray(tokens, np.uint32), np.asarray(options, np.int32)
        a_rows = np.zeros(max(n, 1), np.int32)
        args = capi.InferArgs(C.sizeof(capi.InferArgs), n, capi.ptr(a_slot).value, capi.ptr(a_ntok).value, capi.ptr(a_tok).value,
                              capi.ptr(a_opt).value, capi.ptr(out).value, out.size, capi.ptr(a_rows).value, capi.ptr(score).value,
                              capi.ptr(argmax).value)
        capi.check(capi.lib().b200rwkv_infer_ex(self._h, C.byref(args)), self._h)
        rows, scores, off, soff = [], [], 0, 0
        for i in range(n):
            r = int(a_rows[i])
            rows.append(out[off:off + r])
            off += r
            if options[i] == capi.OPTION_SCORE:
                scores.append((score[soff:soff + ntok[i]], argmax[soff:soff + ntok[i]]))
                soff += ntok[i]
            else:
                scores.append(None)
        return rows, scores

    def infer_snapshots(self, slots, ntok, tokens, options, at, reuse=None):
        """b200rwkv_infer_snapshots: infer_ex(slots, ntok, tokens, options), and one snapshot per (entry, position) of `at`:
        the state of entry's slot after its first `position` tokens of this call, with that token's logits row.  `reuse`:
        None, or one TensorGpu / id / None per snapshot; a given one is overwritten in place.  Returns (rows, scores,
        [TensorGpu]) with rows and scores as infer_ex returns them."""
        V = self.info["num_vocab"]
        n = len(slots)
        total = sum(nt if o == capi.OPTION_FULL else (1 if (o == capi.OPTION_LAST and nt > 0) else 0)
                    for nt, o in zip(ntok, options))
        nscore = sum(nt for nt, o in zip(ntok, options) if o == capi.OPTION_SCORE)
        out = np.empty((max(total, 1), V), np.float32)
        score = np.empty(max(nscore, 1), np.float32)
        argmax = np.empty(max(nscore, 1), np.uint32)
        a_slot, a_ntok = np.asarray(slots, np.int32), np.asarray(ntok, np.int32)
        a_tok, a_opt = np.asarray(tokens, np.uint32), np.asarray(options, np.int32)
        a_rows = np.zeros(max(n, 1), np.int32)
        args = capi.InferArgs(C.sizeof(capi.InferArgs), n, capi.ptr(a_slot).value, capi.ptr(a_ntok).value, capi.ptr(a_tok).value,
                              capi.ptr(a_opt).value, capi.ptr(out).value, out.size, capi.ptr(a_rows).value, capi.ptr(score).value,
                              capi.ptr(argmax).value)
        k = len(at)
        s_entry = np.asarray([e for e, _ in at] or [0], np.int32)
        s_tok = np.asarray([p for _, p in at] or [0], np.int32)
        reuse = list(reuse) if reuse is not None else [None] * k
        if len(reuse) != k:
            raise ValueError(f"reuse holds {len(reuse)} entries for {k} snapshots")
        ids = np.asarray([(r.id if isinstance(r, TensorGpu) else int(r or 0)) for r in reuse] or [0], np.uint64)
        capi.check(capi.lib().b200rwkv_infer_snapshots(self._h, C.byref(args), k, capi.ptr(s_entry), capi.ptr(s_tok),
                                                        capi.ptr(ids)), self._h)
        rows, scores, off, soff = [], [], 0, 0
        for i in range(n):
            r = int(a_rows[i])
            rows.append(out[off:off + r])
            off += r
            if options[i] == capi.OPTION_SCORE:
                scores.append((score[soff:soff + ntok[i]], argmax[soff:soff + ntok[i]]))
                soff += ntok[i]
            else:
                scores.append(None)
        snaps = [r if isinstance(r, TensorGpu) else TensorGpu(self, int(ids[j])) for j, r in enumerate(reuse)]
        return rows, scores, snaps

    # ---- top-n log-probabilities of every scored row (b200rwkv_score_top) ----
    def score_top(self, n: int) -> None:
        """Every following infer_ex / infer_snapshots call also reduces each scored row to its n best (id, log-probability)
        pairs, read with last_score_top(); 0 turns it off."""
        capi.check(capi.lib().b200rwkv_score_top(self._h, int(n)), self._h)
        self._top_n = int(n)

    def last_score_top(self):
        """(ids uint32 [rows][n], log-probabilities f32 [rows][n]) of the most recent infer call, rows = its scored tokens in
        score order."""
        rows = capi.check(capi.lib().b200rwkv_last_score_top(self._h, None, None, 0), self._h)
        ids = np.empty((rows, self._top_n), np.uint32)
        lp = np.empty((rows, self._top_n), np.float32)
        capi.check(capi.lib().b200rwkv_last_score_top(self._h, capi.ptr(ids), capi.ptr(lp), ids.size), self._h)
        return ids, lp

    @contextlib.contextmanager
    def _score_top_as(self, n):
        old = self._top_n
        self.score_top(n)
        try:
            yield
        finally:
            self.score_top(old)

    @staticmethod
    def _split_tops(ntok, options, lists):
        ids, lp = lists
        tops, off = [], 0
        for nt, o in zip(ntok, options):
            if o == capi.OPTION_SCORE:
                tops.append((ids[off:off + nt], lp[off:off + nt]))
                off += nt
            else:
                tops.append(None)
        return tops

    def perplexity(self, slot: int, tokens, head: float | None = None, top_n: int | None = None):
        """The reference's `perplexity()` (run.rs:699-755) on one SCORE call, quirks included: without `head` a token 0 is
        fed first (its own score is not used) and the sum is divided by len(tokens) + 1; with `head` (the probability of
        tokens[0] the caller already holds) the first term is ln(head), the kept row's score of tokens[0] is not used, and the
        divisor is len(tokens).  Run on the slot's current state, which it advances like the reference's Full run does.
        With `top_n` returns (perplexity, (ids [len(tokens)][top_n], log-probabilities [len(tokens)][top_n])): the best
        entries of the row each token was scored from (with `head`, token 0's from the slot's kept row)."""
        tokens = [int(t) for t in tokens]
        fed = tokens if head is not None else [0] + tokens
        if top_n is None:
            _, scores = self.infer_ex([slot], [len(fed)], fed, [capi.OPTION_SCORE])
            return self._perplexity(fed, head, scores[0][0])
        _, scores, tops = self.infer_ex([slot], [len(fed)], fed, [capi.OPTION_SCORE], top_n=top_n)
        k = len(fed) - len(tokens)
        return self._perplexity(fed, head, scores[0][0]), (tops[0][0][k:], tops[0][1][k:])

    @staticmethod
    def _perplexity(fed, head, score) -> float:
        logp = [np.float32(np.log(np.float32(head)))] if head is not None else []
        logp += [np.float32(x) for x in score[1:len(fed)]]
        total = np.float32(0.0)
        for x in logp:                         # `.sum()` over f32 in order, as the iterator does
            total = np.float32(total + x)
        return float(np.float32(-total / np.float32(len(fed))))

    def softmax(self, tensors):
        """`softmax(&context, Vec<TensorCpu<f32>>)`: list of [V] rows in, list out."""
        if not tensors:
            return []
        x = np.ascontiguousarray(np.stack([np.asarray(t, np.float32).reshape(-1) for t in tensors], 0))
        y = np.empty_like(x)
        capi.check(capi.lib().b200rwkv_softmax(self._h, x.shape[0], capi.ptr(x), capi.ptr(y)), self._h)
        return [y[i] for i in range(y.shape[0])]

    def _sample_args(self, slots, penalties, bias, allow):
        """The slot list and adjustment lists of the sampling entries as C arrays: (slots, penalty offsets / tokens / values,
        allow bits or None, bias offsets / tokens / values)."""
        n = len(slots)
        V = self.info["num_vocab"]

        def pack(maps):
            off = np.zeros(n + 1, np.int32)
            toks, vals = [], []
            for i in range(n):
                m = (maps[i] if maps is not None else None) or {}
                toks.extend(int(t) for t in m.keys())
                vals.extend(float(v) for v in m.values())
                off[i + 1] = len(toks)
            return off, np.asarray(toks, np.uint32), np.asarray(vals, np.float32)

        po, pt, pv = pack(penalties)
        bo, bt, bv = pack(bias)
        bits = None
        if allow is not None:
            a = np.asarray(allow, bool).reshape(n, V)
            words = (V + 31) // 32
            padded = np.zeros((n, words * 32), bool)
            padded[:, :V] = a
            bits = np.ascontiguousarray(np.packbits(padded.reshape(n, words, 32), axis=2, bitorder="little").view(np.uint32).reshape(n, words))
        return np.asarray(slots, np.int32), po, pt, pv, bits, bo, bt, bv

    def sample_topk(self, slots, penalties=None, bias=None, allow=None, top_k: int = 128):
        """GPU front half of sampling (b200rwkv_sample_topk): for each slot the `top_k` most probable tokens of its last
        logits row after penalties / grammar mask / bias, as (ids [n, top_k] uint32, probs [n, top_k] f32).
        penalties, bias: per-slot dict token -> value (the reference's HashMaps, nucleus.rs:29, run.rs:679);
        allow: optional [n, V] bool array (tokens the formatter allows)."""
        n = len(slots)
        a_slot, po, pt, pv, bits, bo, bt, bv = self._sample_args(slots, penalties, bias, allow)
        ids = np.empty((n, top_k), np.uint32)
        probs = np.empty((n, top_k), np.float32)
        capi.check(capi.lib().b200rwkv_sample_topk(self._h, n, capi.ptr(a_slot), capi.ptr(po), capi.ptr(pt), capi.ptr(pv),
                                                   capi.ptr(bits) if bits is not None else None, capi.ptr(bo), capi.ptr(bt),
                                                   capi.ptr(bv), top_k, capi.ptr(ids), capi.ptr(probs)), self._h)
        return ids, probs

    def sample_probs(self, slots, penalties=None, bias=None, allow=None) -> np.ndarray:
        """The whole adjusted distribution of each slot's last logits row (b200rwkv_sample_probs): softmax of the row after
        penalties / grammar mask / bias, [n, V] f32 -- what run.rs:673-691 hands to Sampler::sample, for the samplers that
        read every probability (Mirostat, Typical, Nucleus with top_k > 128).  Arguments as sample_topk."""
        n = len(slots)
        a_slot, po, pt, pv, bits, bo, bt, bv = self._sample_args(slots, penalties, bias, allow)
        out = np.empty((n, self.info["num_vocab"]), np.float32)
        capi.check(capi.lib().b200rwkv_sample_probs(self._h, n, capi.ptr(a_slot), capi.ptr(po), capi.ptr(pt), capi.ptr(pv),
                                                    capi.ptr(bits) if bits is not None else None, capi.ptr(bo), capi.ptr(bt),
                                                    capi.ptr(bv), capi.ptr(out)), self._h)
        return out

    def launch_count(self) -> int:
        n = C.c_int64(0)
        capi.check(capi.lib().b200rwkv_launch_count(self._h, C.byref(n)), self._h)
        return n.value

    def keep_hidden(self, enable: bool = True, layers=None) -> None:
        """keep_hidden(bool): record the residual stream after the last layer for every token of each infer call
        (b200rwkv_keep_hidden).  keep_hidden(layers=[...]): record it after each listed layer instead (at most 8 distinct
        layers, b200rwkv_keep_hidden_layers); layers=[] turns that recording off.  The two are independent."""
        if layers is None:
            capi.check(capi.lib().b200rwkv_keep_hidden(self._h, int(enable)), self._h)
            return
        a = np.asarray(layers, np.int32).reshape(-1)
        capi.check(capi.lib().b200rwkv_keep_hidden_layers(self._h, a.size, capi.ptr(a) if a.size else None), self._h)

    def last_hidden(self, max_rows: int = 64, layer: int | None = None) -> np.ndarray:
        """Residual stream per token of the most recent infer call: after the last layer (all tokens after keep_hidden()),
        or after `layer`, which that call must have recorded (keep_hidden(layers=[...]))."""
        Cc = self.info["num_emb"]
        buf = np.empty((max_rows, Cc), np.float32)
        if layer is None:
            r = capi.lib().b200rwkv_last_hidden(self._h, capi.ptr(buf), buf.size)
        else:
            r = capi.lib().b200rwkv_last_hidden_layer(self._h, int(layer), capi.ptr(buf), buf.size)
        capi.check(r, self._h)
        return buf[:r]

    def embed(self, slot: int, tokens, layer: int) -> np.ndarray:
        """The embeddings route (reference docs/doc-api/openai.md:376-437): feed `tokens` to `slot` in one infer call with
        no logits and return the residual stream after `layer` at the last token, [num_emb] f32.  Advances the slot's state;
        turns layer recording off afterwards."""
        tokens = [int(t) for t in tokens]
        if not tokens:
            raise capi.B200Error(capi.ERR_INVALID, "embed: no tokens")
        self.keep_hidden(layers=[layer])
        try:
            self.infer_raw([slot], [len(tokens)], tokens, [capi.OPTION_NONE])
            return self.last_hidden(max_rows=len(tokens), layer=layer)[-1].copy()
        finally:
            self.keep_hidden(layers=[])

    _POOL_MODES = {"last": capi.POOL_LAST, "mean": capi.POOL_MEAN}

    def bind_adapter(self, slots, ids) -> None:
        """Slot slots[i] runs adapter ids[i] (1..n of the `adapters` list, 0 = the base model) from the next infer call on
        (b200rwkv_bind_adapter)."""
        slots = np.ascontiguousarray(slots, dtype=np.int32)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        if slots.shape != ids.shape:
            raise capi.B200Error(capi.ERR_INVALID, "bind_adapter: slots and ids differ in length")
        capi.check(capi.lib().b200rwkv_bind_adapter(self._h, slots.size, capi.ptr(slots), capi.ptr(ids)), self._h)

    def load_adapter(self, id: int, st, alpha: float) -> None:
        """Fills the empty adapter place `id` with the adapter file `st` at `alpha` (b200rwkv_load_adapter)."""
        img = np.ascontiguousarray(st, dtype=np.uint8)
        capi.check(capi.lib().b200rwkv_load_adapter(self._h, int(id), capi.ptr(img), img.size, float(alpha)), self._h)

    def unload_adapter(self, id: int) -> None:
        """Empties adapter place `id`; no slot may be bound to it (b200rwkv_unload_adapter)."""
        capi.check(capi.lib().b200rwkv_unload_adapter(self._h, int(id)), self._h)

    def update_weights(self, st) -> None:
        """Replaces the tensors the safetensors image `st` holds (any subset of the model's) in place
        (b200rwkv_update_weights).  Afterwards the engine computes what one created from the updated image would; slot
        states, snapshots and kept rows still hold what the old weights computed."""
        img = np.ascontiguousarray(st, dtype=np.uint8)
        capi.check(capi.lib().b200rwkv_update_weights(self._h, capi.ptr(img), img.size), self._h)

    def head_format(self, kind) -> None:
        """The vocabulary head's weight format from the next infer call on (b200rwkv_head_format): "None" (f16, the default),
        "Int8", "NF4", "FP8" or "Int4", or a capi.QUANT_* value -- head.weight through the quantiser of quantised layers.
        "None" returns to the f16 head bit for bit; slot states, snapshots and kept rows keep what the old head computed."""
        capi.check(capi.lib().b200rwkv_head_format(self._h, quant_kind(kind, "head_format")), self._h)

    def update_weights_from_tensors(self, tensors: dict) -> None:
        """update_weights from torch tensors on the engine's device: {name: contiguous CUDA tensor} in float16, bfloat16 or
        float32, each in the model's shape, rounded to F16 on the device (b200rwkv_update_weights_device)."""
        import torch
        kinds = {torch.float16: capi.DTYPE_F16, torch.bfloat16: capi.DTYPE_BF16, torch.float32: capi.DTYPE_F32}
        if not tensors:
            raise capi.B200Error(capi.ERR_INVALID, "update_weights_from_tensors: no tensors")
        table = (capi.WeightSrc * len(tensors))()
        names = []
        for i, (name, t) in enumerate(tensors.items()):
            if not isinstance(t, torch.Tensor) or not t.is_cuda or not t.is_contiguous() or t.dtype not in kinds:
                raise capi.B200Error(capi.ERR_INVALID, f"update_weights_from_tensors: {name} must be a contiguous CUDA tensor "
                                                       "in float16, bfloat16 or float32")
            names.append(name.encode())
            table[i].name, table[i].dtype, table[i].data = names[-1], kinds[t.dtype], t.data_ptr()
        torch.cuda.synchronize(next(iter(tensors.values())).device)     # the producers' writes have landed
        capi.check(capi.lib().b200rwkv_update_weights_device(self._h, len(tensors), table), self._h)

    def keep_hidden_pooled(self, layers, mode="last") -> None:
        """Reduce the residual stream after each listed layer to one row per entry of every following infer call
        (b200rwkv_keep_hidden_pooled): mode "last" keeps the row of the entry's last token, "mean" the f32 mean of its rows
        in token order (capi.POOL_LAST / POOL_MEAN are accepted too).  At most 8 distinct layers; layers=[] turns it off.
        Independent of keep_hidden."""
        a = np.asarray(layers, np.int32).reshape(-1)
        capi.check(capi.lib().b200rwkv_keep_hidden_pooled(self._h, a.size, capi.ptr(a) if a.size else None,
                                                          self._POOL_MODES.get(mode, mode)), self._h)

    def last_hidden_pooled(self, layer: int, max_rows: int | None = None):
        """The pooled rows of the most recent infer call after `layer`, which that call must have pooled: (rows [n, num_emb]
        f32 in entry order, token counts [n] int32).  max_rows: an upper bound on the call's entries (default max_batch)."""
        rows = self.max_batch if max_rows is None else max_rows
        buf = np.empty((max(rows, 1), self.info["num_emb"]), np.float32)
        ntok = np.zeros(max(rows, 1), np.int32)
        r = capi.lib().b200rwkv_last_hidden_pooled(self._h, int(layer), capi.ptr(buf), rows * buf.shape[1], capi.ptr(ntok))
        capi.check(r, self._h)
        return buf[:r], ntok[:r]

    def embed_many(self, slots, token_lists, layer: int, mode="last") -> np.ndarray:
        """The embeddings route for several inputs at once: feed token_lists[i] to slots[i] in one infer call with no logits
        and return the pooled residual stream after `layer`, [n, num_emb] f32.  Only num_emb floats per input leave the
        device.  Advances the slots' states; turns pooling off afterwards."""
        token_lists = [[int(t) for t in toks] for toks in token_lists]
        if len(token_lists) != len(slots) or not all(token_lists):
            raise capi.B200Error(capi.ERR_INVALID, "embed_many: one non-empty token list per slot")
        self.keep_hidden_pooled([layer], mode)
        try:
            self.infer_raw(list(slots), [len(t) for t in token_lists], sum(token_lists, []), [capi.OPTION_NONE] * len(slots))
            return self.last_hidden_pooled(layer, max_rows=len(slots))[0].copy()
        finally:
            self.keep_hidden_pooled([])

    def debug_read(self, name: str, rows: int = 64) -> np.ndarray:
        buf = np.empty(rows * 65536, np.float32)
        cols = capi.lib().b200rwkv_debug_read(self._h, name.encode(), capi.ptr(buf), buf.size)
        capi.check(cols, self._h)
        return buf[: rows * cols].reshape(rows, cols)

    def debug_fills(self, name: str) -> list[tuple[dict, dict]]:
        """Test aid: every weight fill the engine runs for tensor `name` (b200rwkv_debug_fill), read back from the device, as
        (info, parts).  info: the b200rwkv_fill_info fields.  parts, R = tiles * 128 rows and Kp = kb * 128 columns, padding
        included: SEG "w" f16 bits [R, Kp] (qtype NONE) or "codes" u8 [R, Kp] with Int8 / Int4 "min" and "scale" f16 [R, kb],
        NF4 "absmax" f16 [R, 2 kb], FP8 "scale" f32 [R]; a W' segment also "tail" f16 bits [R, ad_tail * 128].  VEC / DECAY
        "v" f32 [count], RAW "v" f16 bits [count], FOLD "v" f16 bits [N, K, 64], INIT "v" f32 [head_size + 2, num_emb]."""
        lib, out = capi.lib(), []
        for i in range(capi.check(lib.b200rwkv_debug_fills(self._h, name.encode()), self._h)):
            fi = capi.FillInfo()
            capi.check(lib.b200rwkv_debug_fill(self._h, name.encode(), i, C.byref(fi), None, 0), self._h)
            raw = np.empty(fi.bytes, np.uint8)
            capi.check(lib.b200rwkv_debug_fill(self._h, name.encode(), i, C.byref(fi), capi.ptr(raw), raw.size), self._h)
            info = fi.as_dict()
            out.append((info, _fill_parts(info, raw, self.info["head_size"], self.info["num_emb"])))
        return out

    def bench_decode(self, slots, tokens: np.ndarray, warmup: int, steps: int, flush_l2: bool = False):
        a_slot = np.asarray(slots, np.int32)
        tok = np.ascontiguousarray(tokens, dtype=np.uint32)
        assert tok.size == (warmup + steps) * len(slots)
        ms = C.c_float(0)
        launches = C.c_int64(0)
        self.step_ms = np.zeros(steps, np.float32)          # CUDA-event time of every timed step (distribution)
        capi.check(capi.lib().b200rwkv_bench_decode(self._h, len(slots), capi.ptr(a_slot), capi.ptr(tok), warmup, steps,
                                                    int(flush_l2), C.byref(ms), C.byref(launches), capi.ptr(self.step_ms)), self._h)
        return ms.value, launches.value

    def profile_insitu(self, slots, tokens, reps: int = 5):
        """Per-launch windows of one graph-replayed decode step (b200rwkv_profile_insitu): list of dicts + step_us."""
        a_slot = np.asarray(slots, np.int32)
        tok = np.ascontiguousarray(tokens, dtype=np.uint32)
        cap = 1024
        n = C.c_int32(0)
        types = np.zeros(cap, np.int32)
        st, en = np.zeros(cap, np.float64), np.zeros(cap, np.float64)
        by = np.zeros(cap, np.int64)
        step = C.c_double(0)
        capi.check(capi.lib().b200rwkv_profile_insitu(self._h, len(slots), capi.ptr(a_slot), capi.ptr(tok), reps, cap, C.byref(n),
                                                      capi.ptr(types), capi.ptr(st), capi.ptr(en), capi.ptr(by), C.byref(step)), self._h)
        k = n.value
        return [{"type": int(types[i]), "start_us": float(st[i]), "end_us": float(en[i]), "bytes": int(by[i])} for i in range(k)], step.value

    def profile_step(self, slots, tokens):
        a_slot = np.asarray(slots, np.int32)
        tok = np.ascontiguousarray(tokens, dtype=np.uint32)
        ms = (C.c_float * 4)()
        ln = (C.c_int32 * 4)()
        wb = C.c_int64(0)
        capi.check(capi.lib().b200rwkv_profile_step(self._h, len(slots), capi.ptr(a_slot), capi.ptr(tok), C.byref(ms),
                                                    C.byref(ln), C.byref(wb)), self._h)
        return list(ms), list(ln), wb.value
