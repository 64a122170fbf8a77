"""Every weight buffer an engine builds, read back with b200rwkv_debug_fill and compared bit for bit with references built
from the image alone (O.parse_st) and the committed oracles: oracle/quant_numpy.py, tests/fp8_oracle.py, tests/int4_oracle.py
and test_gpu_load_kernels' LoRA blend and f16 -> f32 references.

The checks through arithmetic (logits at 1e-3, the GEMM and step-stage bounds) cannot see a few wrong codes: one Int8 code
off by one in a block of a K = 4096 row moves an output by about 0.13 of the GEMM bound.  Here every code, parameter,
padding element and adapter tail block is pinned:
  - SEG fills (projection plans): f16 plans hold the matrix's bits; quantised plans hold the oracle's codes and parameters of
    the WHOLE matrix, cut to the fill's rows and columns (so an FP8 slice's row scale is the whole row's).  Padding rows
    (n >= N) and columns (k >= K) are exact zeros (f16) or dequantise to exact zeros (codes).
  - Coverage: per plan, a matrix's SEG regions tile [0, N) x [0, K) exactly once; one base plan per matrix, at most one W'
    plan (always one for an adapted matrix), and one more fill for a quantised head.  att.output and ffn.value are cut into
    the split-K factor test_gpu_gemm.pick_split gives.
  - W' plans: the base part equals the base plan's bits; the adapter tail blocks hold f16(f32(alpha) * lora.1) in the
    columns below each adapter's rank and zeros elsewhere (empty places: zeros).
  - VEC fills are one fma of f32(x) with the conversion the model definition needs (vec_conv, from oracle/rwkv_numpy.py),
    DECAY fills within test_gpu_load_kernels' bound, RAW fills the tensor's bits, FOLD fills the k-major transpose, INIT fills
    the State::init rows.
  - Tensor-parallel ranks (b200rwkv_create_tp, never connected): a split matrix holds each cell on exactly one rank, a copied
    matrix on every rank (TP_CUTS names which is which).
No configuration runs a model step.
"""
import dataclasses

import numpy as np
import pytest

import fp8_oracle as F8
import int4_oracle as I4
import test_gpu_gemm as G
from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O
from test_gpu_load_kernels import fma_f32, lora_ref
from test_gpu_load_kernels import pick_split as tp_pick_split

pytestmark = pytest.mark.gpu
f16, f32, f64 = np.float16, np.float32, np.float64
NONE, INT8, NF4, FP8, INT4 = capi.QUANT_NONE, capi.QUANT_INT8, capi.QUANT_NF4, capi.QUANT_FP8, capi.QUANT_INT4
FORMATS = [NONE, INT8, NF4, FP8, INT4]
FMT_NAME = {NONE: "f16", INT8: "int8", NF4: "nf4", FP8: "fp8", INT4: "int4"}
BASE, ADAPTER, HEAD = capi.PLAN_BASE, capi.PLAN_ADAPTER, capi.PLAN_HEAD


def u16(a):
    return np.ascontiguousarray(a).view(np.uint16)


def cdiv(a, b):
    return -(-a // b)


# ---- references ----

def quantize(qt, M):
    """The oracle's codes and parameters of a whole [N, K] f16 matrix, named as runtime.Model.debug_fills names them."""
    if qt == INT8:
        q, mn, mx = Q.quant_int8(M)
        return {"codes": q, "min": mn, "scale": Q.int8_scale(mn, mx)}
    if qt == NF4:
        q, am = Q.quant_nf4(M)
        return {"codes": q, "absmax": am}
    if qt == FP8:
        q, s = F8.quant_fp8(M)
        return {"codes": q, "scale": s}
    q, mn, s = I4.quant_int4(M)
    return {"codes": q, "min": mn, "scale": s}


PARAM_BLOCK = {INT8: 128, INT4: 128, NF4: 64}       # inputs per block parameter (FP8: one scale per row)


def dequantize(qt, p):
    """float64 weights of read-back codes and parameters (padding included)."""
    c = p["codes"].astype(f64)
    if qt == FP8:
        return F8.e4m3_decode(p["codes"]).astype(f64) * p["scale"].astype(f64)[:, None]
    if qt == NF4:
        return Q.NF4_LEVELS.astype(f64)[p["codes"]] * np.repeat(p["absmax"].astype(f64), 64, axis=1)
    return c * np.repeat(p["scale"].astype(f64), 128, axis=1) + np.repeat(p["min"].astype(f64), 128, axis=1)


def decay_bound(x64):
    """test_gpu_load_kernels.test_decay_table_within_the_derived_bound's bound on expf(-expf(x)) against float64."""
    with np.errstate(over="ignore", invalid="ignore"):
        ex = np.exp(x64)
        z = np.exp(-ex)
        D = 2.0 ** -22 * ex + 2.0 ** -148
        bound = (1 + 2.0 ** -22) * (np.exp(D - ex) - z) + 2.0 ** -22 * z + 2.0 ** -148 + 2.0 ** -50 * (1 + ex) * z
    return z, np.where(np.isfinite(ex), bound, 2.0 ** -148)


# Conversion of each f32 vector (scale, bias of one fma), from oracle/rwkv_numpy.py: RWKV-5's token-shift mixes enter as
# 1 - mu (x_* = xx + (prev - xx)(1 - mu)); every other vector as stored.
def vec_conv(version, name):
    if version == 5 and (".att.time_mix_" in name or ".ffn.time_mix_" in name):
        return -1.0, 1.0
    return 1.0, 0.0


# per-channel vectors a tensor-parallel rank holds only its [rank Cl, (rank + 1) Cl) part of
RANK_VECTORS = (".att.ln_x.weight", ".att.ln_x.bias", ".att.time_first", ".att.w0", ".att.a0", ".att.v0", ".att.k_k",
                ".att.k_a", ".att.r_k")


def rank_vector(version, name):
    return name.endswith(RANK_VECTORS) or (version == 6 and name.endswith(".att.time_decay"))


# How tensor parallelism cuts each projection matrix: "rows" (column parallel: a rank holds rows [r n / W, (r + 1) n / W)),
# "cols" (row parallel: columns [r k / W, (r + 1) k / W), each cut again into split-K slices), "copy" (every rank holds all).
TP_CUTS = {
    5: {"att.receptance": "rows", "att.key": "rows", "att.value": "rows", "att.gate": "rows", "att.output": "cols",
        "ffn.key": "rows", "ffn.receptance": "rows", "ffn.value": "cols"},
    6: {"att.receptance": "rows", "att.key": "rows", "att.value": "rows", "att.gate": "rows", "att.output": "cols",
        "ffn.key": "rows", "ffn.receptance": "rows", "ffn.value": "cols", "att.time_mix_w1": "copy", "att.time_mix_w2": "copy",
        "att.time_decay_w1": "copy", "att.time_decay_w2": "rows"},
    7: {"att.receptance": "rows", "att.key": "rows", "att.value": "rows", "att.output": "cols", "ffn.key": "rows",
        "ffn.value": "cols", "att.w1": "copy", "att.a1": "copy", "att.v1": "copy", "att.g1": "copy", "att.w2": "rows",
        "att.a2": "rows", "att.v2": "rows", "att.g2": "rows"},
}


def kind_of(name):
    """'att.key' of 'blocks.3.att.key.weight', 'head' of 'head.weight'."""
    if not name.startswith("blocks."):
        return name[:-len(".weight")] if name.endswith(".weight") else name
    k = name.split(".", 2)[2]
    return k[:-len(".weight")] if k.endswith(".weight") else k


def layer_of(name):
    return int(name.split(".")[1]) if name.startswith("blocks.") else -1


def seg_tensors(shape, w):
    """The tensors the engine runs as projection segments: every 2-D `.weight` but the embedding, the RWKV-6 ddlerp and decay
    LoRA matrices (time_decay_w2 only when its rank is above 128: below, the WKV kernel folds it), RWKV-7's LoRA matrices
    (v1 / v2 from layer 1 on)."""
    out = set()
    for n, a in w.items():
        k, l = kind_of(n), layer_of(n)
        if n.endswith(".weight") and a.ndim == 2 and n != "emb.weight":
            out.add(n)
        elif shape.version == 6 and k in ("att.time_mix_w1", "att.time_mix_w2", "att.time_decay_w1"):
            out.add(n)
        elif shape.version == 6 and k == "att.time_decay_w2" and shape.Dd > 128:
            out.add(n)
        elif shape.version == 7 and k in ("att.w1", "att.w2", "att.a1", "att.a2", "att.g1", "att.g2"):
            out.add(n)
        elif shape.version == 7 and k in ("att.v1", "att.v2") and l > 0:
            out.add(n)
    return out


@dataclasses.dataclass
class Config:
    shape: synth.Shape
    w: dict                             # name -> the values the engine must hold (after load-time LoRA blends)
    quant_layers: int = 0
    qtype: int = NONE
    head_qt: int = NONE
    places: int = 0                     # adapter places (0: no adapters)
    held: list = dataclasses.field(default_factory=list)        # per place: (lora tensors, alpha), or None while empty
    adapted: set = dataclasses.field(default_factory=set)       # matrices whose W' plan carries adapter tail blocks
    rank: int = 0
    world: int = 1


class Checker:
    def __init__(self, cfg: Config):
        self.cfg = cfg
        self._oracle = {}
        self.holdings = {}              # tensor parallel: name -> per-cell count of ranks holding it

    def matrix(self, name, off, rows, ld):
        return self.cfg.w[name].reshape(-1)[off:off + rows * ld].reshape(rows, ld)

    def oracle(self, name, off, M, qt):
        key = (name, off, qt)
        if key not in self._oracle:
            self._oracle[key] = quantize(qt, np.ascontiguousarray(M))
        return self._oracle[key]

    def expect_qt(self, name, plan):
        c = self.cfg
        if plan == HEAD:
            return c.head_qt
        if c.qtype != NONE and 0 <= layer_of(name) < c.quant_layers and kind_of(name) + ".weight" in Q.QUANT_MATRICES:
            return c.qtype
        return NONE

    # ---- one fill ----
    def check_seg(self, name, i, info, parts):
        c = self.cfg
        what = f"{name} fill {i} (plan {info['plan']}, rows {info['n0']}+{info['N']}, cols {info['k0']}+{info['K']})"
        shape = c.w[name].shape
        rows, ld = (shape[1], shape[2]) if len(shape) == 3 else shape
        assert info["ld"] == ld and info["off"] % (rows * ld) == 0, what
        n0, N, k0, K = info["n0"], info["N"], info["k0"], info["K"]
        assert 0 <= n0 and n0 + N <= rows and 0 <= k0 and k0 + K <= ld and N > 0 and K > 0, what
        assert info["tiles"] == cdiv(N, 128) and info["kb"] == cdiv(K, 128), what
        qt = self.expect_qt(name, info["plan"])
        assert info["qtype"] == qt, what
        M = self.matrix(name, info["off"], rows, ld)
        R, Kp = info["tiles"] * 128, info["kb"] * 128
        if qt == NONE:
            want = np.zeros((R, Kp), np.uint16)
            want[:N, :K] = u16(M)[n0:n0 + N, k0:k0 + K]
            bad = parts["w"] != want
            assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} f16 elements differ, first at {np.argwhere(bad)[0]}"
        else:
            o = self.oracle(name, info["off"], M, qt)
            bad = parts["codes"][:N, :K] != o["codes"][n0:n0 + N, k0:k0 + K]
            assert not bad.any(), f"{what}: {int(bad.sum())} codes differ from the oracle, first at {np.argwhere(bad)[0]}"
            if qt == FP8:
                assert np.array_equal(parts["scale"][:N].view(np.uint32), o["scale"][n0:n0 + N].view(np.uint32)), \
                    f"{what}: row scales differ from the whole rows' (first row {np.argwhere(parts['scale'][:N] != o['scale'][n0:n0 + N])[:1]})"
            else:
                b = PARAM_BLOCK[qt]
                for p in ("min", "scale", "absmax"):
                    if p in o:
                        bad = u16(parts[p][:N, :K // b]) != u16(o[p][n0:n0 + N, k0 // b:(k0 + K) // b])
                        assert not bad.any(), f"{what}: {int(bad.sum())} block {p} values differ, first at {np.argwhere(bad)[0]}"
            assert K == Kp, what                # quantised K is whole 128-input blocks: the padding is rows N..R
            deq = dequantize(qt, {k: v[N:] for k, v in parts.items() if k != "tail"})
            assert np.all(deq == 0), f"{what}: padding rows do not dequantise to zeros"
        self.check_tail(name, what, info, parts)

    def check_tail(self, name, what, info, parts):
        c = self.cfg
        ad = info["plan"] == ADAPTER and name in c.adapted and info["k0"] + info["K"] == info["ld"]
        assert info["ad_tail"] == (c.places if ad else 0), what
        if not ad:
            return
        n0, N, R = info["n0"], info["N"], info["tiles"] * 128
        want = np.zeros((R, c.places * 128), np.uint16)
        base = name[:-len(".weight")]
        for a, h in enumerate(c.held):
            if h is None or base + ".lora.1" not in h[0]:
                continue
            b = h[0][base + ".lora.1"]
            r = b.shape[1]
            want[:N, a * 128:a * 128 + r] = u16((f32(h[1]) * b[n0:n0 + N].astype(f32)).astype(f16))
        bad = parts["tail"] != want
        assert not bad.any(), f"{what}: {int(bad.sum())} adapter tail elements differ, first at {np.argwhere(bad)[0]}"

    def check_other(self, name, i, info, parts):
        c, s = self.cfg, self.cfg.shape
        what = f"{name} fill {i} (kind {info['kind']})"
        x = c.w[name].reshape(-1)
        Cl = s.C // c.world
        v = parts["v"]
        if info["kind"] in (capi.FILL_VEC, capi.FILL_DECAY):
            off, count = (c.rank * Cl, Cl) if (rank_vector(s.version, name) or info["kind"] == capi.FILL_DECAY) else (0, s.C)
            assert (info["off"], info["count"]) == (off, count), what
            src = x[off:off + count]
            if info["kind"] == capi.FILL_VEC:
                scale, bias = vec_conv(s.version, name)
                want = fma_f32(src.astype(f32), f32(scale), f32(bias))
                assert np.array_equal(v.view(np.uint32), want.view(np.uint32)), f"{what}: {int((v != want).sum())} values differ"
            else:
                assert s.version == 5 and kind_of(name) == "att.time_decay", what
                z, bound = decay_bound(src.astype(f64))
                assert np.all(np.abs(v.astype(f64) - z) <= bound), what
        elif info["kind"] == capi.FILL_RAW:
            assert name == "emb.weight" or (s.version == 6 and kind_of(name) in ("att.time_mix_w1", "att.time_mix_w2")), what
            assert np.array_equal(v, u16(x)), what
        elif info["kind"] == capi.FILL_FOLD:
            assert kind_of(name) == "att.time_decay_w2" and s.Dd <= 128, what
            Hl = s.H // c.world
            w2 = u16(c.w[name])[c.rank * Cl:(c.rank + 1) * Cl]
            assert (info["n0"], info["N"], info["K"]) == (c.rank * Cl, Hl, s.Dd), what
            assert np.array_equal(v, w2.reshape(Hl, 64, s.Dd).transpose(0, 2, 1)), what
        else:
            assert info["kind"] == capi.FILL_INIT and kind_of(name) == "att.time_state", what
            ts = c.w[name].astype(f32)
            want = np.zeros((s.N + 2, s.C), f32)
            want[1:s.N + 1] = ts.transpose(1, 0, 2).reshape(s.N, s.C)
            assert info["n0"] == layer_of(name) and np.array_equal(v, want), what

    # ---- one engine ----
    def check(self, m, names=None):
        c, s = self.cfg, self.cfg.shape
        segs = seg_tensors(s, c.w)
        names = sorted(c.w) if names is None else names
        for name in names:
            fills = m.debug_fills(name)
            by_plan = {}
            for i, (info, parts) in enumerate(fills):
                if info["kind"] == capi.FILL_SEG:
                    self.check_seg(name, i, info, parts)
                    by_plan.setdefault(info["plan"], []).append((info, parts))
                else:
                    self.check_other(name, i, info, parts)
            if name in segs:
                self.check_plans(name, by_plan)
            else:
                assert not by_plan, f"{name} is not a projection matrix, yet has SEG fills"

    def check_plans(self, name, by_plan):
        c, s = self.cfg, self.cfg.shape
        assert BASE in by_plan, f"{name} has no base plan"
        if name in c.adapted:
            assert ADAPTER in by_plan, f"{name} is adapted but has no W' plan"
        if not c.places:
            assert ADAPTER not in by_plan, f"{name} has a W' plan on an engine without adapters"
        assert (HEAD in by_plan) == (name == "head.weight" and c.head_qt != NONE), name
        shape = c.w[name].shape
        rows, ld = (shape[1], shape[2]) if len(shape) == 3 else shape
        nslice = shape[0] if len(shape) == 3 else 1
        for plan, fl in by_plan.items():
            # every plan covers its cut of the matrix once: the whole matrix on one GPU, a rank's cut with tensor parallelism
            cover = np.zeros((nslice, rows, ld), np.int8)
            for info, _ in fl:
                cover[info["off"] // (rows * ld), info["n0"]:info["n0"] + info["N"], info["k0"]:info["k0"] + info["K"]] += 1
            if c.world == 1:
                assert np.all(cover == 1), f"{name} plan {plan}: cells held {cover.min()}..{cover.max()} times"
            else:
                assert cover.max() == 1, f"{name} plan {plan}: a cell held twice"
                if plan == BASE:
                    self.holdings.setdefault(name, np.zeros_like(cover, dtype=np.int16))
                    self.holdings[name] += cover
            if plan == BASE and kind_of(name) in ("att.output", "ffn.value"):
                Kl = ld // c.world
                S = tp_pick_split(Kl, cdiv(rows, 128), c.world, G.num_sms()) if c.world > 1 else G.pick_split(Kl, cdiv(rows, 128))
                assert sorted(i["k0"] for i, _ in fl) == [c.rank * Kl + j * (Kl // S) for j in range(S)], (name, S)
            if plan == ADAPTER:
                # the W' copy holds the base plan's codes
                base = {(i["off"], i["n0"], i["k0"]): p for i, p in by_plan[BASE]}
                for info, parts in fl:
                    b = base[(info["off"], info["n0"], info["k0"])]
                    for k in b:
                        assert np.array_equal(parts[k], b[k]), f"{name}: the W' plan's {k} differ from the base plan's"


# ---- configurations ----

_images = {}


def image(shape, seed=0):
    key = (dataclasses.astuple(shape), seed)
    if key not in _images:
        _images[key] = synth.make_st(shape, seed)
    return _images[key]


def check_engine(shape, quant_layers=0, qtype=NONE, **kw):
    st = image(shape)
    w = O.parse_st(st)
    q = dict(quant=quant_layers, quant_type=qtype) if qtype != NONE else {}
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, **q, **kw)
    try:
        Checker(Config(shape, w, quant_layers if qtype != NONE else 0, qtype)).check(m)
    finally:
        m.close()


PRESETS = ["tiny5", "tiny6", "tiny7", "small6", "small7"]


@pytest.mark.parametrize("qt", FORMATS, ids=[FMT_NAME[q] for q in FORMATS])
@pytest.mark.parametrize("preset", PRESETS)
def test_layers_in_every_format(preset, qt):
    """Every fill of the small models, f16 or with quantised layers (small6: the first 2 of 4 layers)."""
    s = synth.PRESETS[preset]
    check_engine(s, 2 if preset == "small6" else s.L, qt)


def one_layer(preset):
    return dataclasses.replace(synth.PRESETS[preset], L=1, V=4096)


@pytest.mark.parametrize("qt", FORMATS, ids=[FMT_NAME[q] for q in FORMATS])
@pytest.mark.parametrize("preset", ["v6-7b", "v6-3b", "v7-2b9"])
def test_full_size_layer(preset, qt):
    """One layer at the full-size shapes: the split-K slices of att.output and ffn.value (k0 != 0, ld != K), with FP8 row
    scales taken over the whole rows."""
    check_engine(one_layer(preset), 1, qt)


def test_embedding_not_a_multiple_of_128():
    """num_emb 320: K padded up to whole 128-column blocks with zeros (f16 only: quantised layers refuse it)."""
    check_engine(dataclasses.replace(synth.PRESETS["small6"], C=320, F=1120), 0, NONE)


def test_state_tuned_model():
    check_engine(dataclasses.replace(synth.PRESETS["tiny6"], time_state=True), 0, NONE)


@pytest.mark.parametrize("qt", [NONE, INT8, FP8, INT4], ids=["f16", "int8", "fp8", "int4"])
def test_load_time_lora(qt):
    """Two LoRA files blended at load, one after the other, then quantised: the references are test_gpu_load_kernels.lora_ref
    chained, then the oracle."""
    s = synth.PRESETS["tiny6"]
    st = image(s)
    files = [(synth.make_lora_st(s, 8, 1), 0.75), (synth.make_lora_st(s, 16, 2, targets=("att.receptance", "ffn.key")), -1.5)]
    w = dict(O.parse_st(st))
    for img, alpha in files:
        lo = O.parse_st(img)
        for n in list(w):
            base = n[:-len(".weight")]
            if n.endswith(".weight") and base + ".lora.0" in lo:
                w[n] = lora_ref(w[n], lo[base + ".lora.1"], lo[base + ".lora.0"], alpha)
    q = dict(quant=s.L, quant_type=qt) if qt != NONE else {}
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, lora=files, **q)
    try:
        Checker(Config(s, w, s.L if qt != NONE else 0, qt)).check(m)
    finally:
        m.close()


def adapted_matrices(w, files):
    return {n for n in w if n.endswith(".weight") and any(n[:-len(".weight")] + ".lora.0" in f for f in files)}


@pytest.mark.parametrize("preset,qt", [("tiny6", NONE), ("tiny7", INT4), ("tiny5", FP8), ("small6", INT8), ("tiny6", NF4)])
def test_adapters(preset, qt):
    """b200rwkv_create_adapters (quant_adapters with quantised layers): W' plans hold the base plan's bits and f16(alpha B)
    tail blocks, one per adapter; other adapters' blocks and columns past a rank are zero."""
    s = synth.PRESETS[preset]
    st = image(s)
    w = O.parse_st(st)
    imgs = [(synth.make_lora_st(s, 8, 3), 0.1), (synth.make_lora_st(s, 5, 4, targets=("att.value", "ffn.value")), -0.37)]
    los = [O.parse_st(i) for i, _ in imgs]
    q = dict(quant=2, quant_type=qt, quant_adapters=True) if qt != NONE else {}
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, adapters=imgs, **q)
    try:
        cfg = Config(s, w, 2 if qt != NONE else 0, qt, places=2, held=[(lo, a) for lo, (_, a) in zip(los, imgs)],
                     adapted=adapted_matrices(w, los))
        Checker(cfg).check(m)
    finally:
        m.close()


@pytest.mark.parametrize("preset,qt", [("tiny6", NONE), ("tiny7", FP8), ("small6", INT4)])
def test_adapter_places(preset, qt):
    """b200rwkv_create_adapter_places with quant_adapters: every targeted matrix has a W' plan whose tails are zero while the
    places are empty, hold the adapter after load_adapter, and are zero again after unload_adapter."""
    s = synth.PRESETS[preset]
    st = image(s)
    w = O.parse_st(st)
    targets = list(capi.TARGETS)
    q = dict(quant=2, quant_type=qt, quant_adapters=True) if qt != NONE else {}
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, adapter_places=2, adapter_targets=targets, **q)
    adapted = {n for n in w if n.endswith(".weight") and (kind_of(n) in capi.TARGETS)}
    img = synth.make_lora_st(s, 12, 5, targets=("att.key", "att.output", "ffn.value"))
    lo = O.parse_st(img)
    names = sorted(seg_tensors(s, w))

    def check(held):
        Checker(Config(s, w, 2 if qt != NONE else 0, qt, places=2, held=held, adapted=adapted)).check(m, names)

    try:
        check([None, None])
        m.load_adapter(2, img, -0.37)
        check([None, (lo, -0.37)])
        m.unload_adapter(2)
        check([None, None])
    finally:
        m.close()


@pytest.mark.parametrize("V", [509, 4096, 65536, 70003])
def test_head_formats(V):
    """Every head format in turn, then NONE again: the quantised head's codes are the oracle's of head.weight, and the f16
    head is untouched throughout."""
    s = dataclasses.replace(synth.PRESETS["tiny6"], V=V)
    st = image(s)
    w = O.parse_st(st)
    m = runtime.Model(st, max_batch=2, token_chunk_size=16)
    try:
        for hq in (INT8, NF4, FP8, INT4, NONE):
            m.head_format(hq)
            cfg = Config(s, w, head_qt=hq)
            Checker(cfg).check(m, ["head.weight"])
            n_fills = len(m.debug_fills("head.weight"))
            assert n_fills == (1 if hq == NONE else 2), (hq, n_fills)
    finally:
        m.close()


def test_update_weights_from_an_image():
    """update_weights with a whole second image on an engine with Int8 layers and an FP8 head: every fill holds the new
    values, the head's codes included."""
    s = synth.PRESETS["small6"]
    st, st2 = image(s), image(s, 1)
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, quant=2, quant_type=INT8)
    try:
        m.head_format(FP8)
        m.update_weights(st2)
        Checker(Config(s, O.parse_st(st2), 2, INT8, head_qt=FP8)).check(m)
    finally:
        m.close()


def tie_values(rng, shape, dtype):
    """Values whose f16 rounding is a tie on about half the elements: f16 midpoints (F32), or odd multiples of 2^-25, which
    bf16 holds exactly and f16 cannot (BF16); the rest ordinary values."""
    import torch
    base = (rng.standard_normal(shape) * 0.05).astype(f16)
    if dtype == torch.float32:
        up = np.nextafter(base, f16(np.inf))
        mid = ((base.astype(f64) + up.astype(f64)) / 2).astype(f32)
        assert np.array_equal(mid.astype(f64), (base.astype(f64) + up.astype(f64)) / 2)
        x = np.where(rng.integers(0, 2, shape).astype(bool), mid, base.astype(f32))
    else:
        # base values cut to bf16's 8 significant bits (f16 holds them); ties: odd multiples of 2^-25 (f16's subnormal step
        # is 2^-24)
        b16 = (base.astype(f32).view(np.uint32) & np.uint32(0xFFFF0000)).view(f32)
        odd = (2 * rng.integers(-127, 128, shape) + 1).astype(f64) * 2.0 ** -25
        x = np.where(rng.integers(0, 2, shape).astype(bool), odd, b16.astype(f64)).astype(f32)
    t = torch.from_numpy(np.ascontiguousarray(x)).to(dtype)
    assert np.array_equal(t.float().numpy(), x)                 # exact in the source type
    return t, x.astype(f16)                                     # numpy: round to nearest, ties to even


@pytest.mark.parametrize("dt", ["float16", "bfloat16", "float32"])
def test_update_weights_from_device_tensors(dt):
    """update_weights_from_tensors with F16, BF16 and F32 tensors on values that are f16 rounding ties: the engine's fills
    hold numpy's round-to-nearest-even f16 values, through quantised and f16 layers, vectors, the embedding and the head."""
    import torch
    dtype = getattr(torch, dt)
    s = synth.PRESETS["tiny6"]
    st = image(s)
    w = dict(O.parse_st(st))
    rng = np.random.default_rng(17)
    names = ["blocks.0.att.key.weight", "blocks.1.ffn.value.weight", "blocks.1.att.time_mix_w2", "blocks.0.ln1.weight",
             "blocks.1.att.time_decay_w2", "emb.weight", "head.weight"]
    tensors = {}
    for n in names:
        t, want = tie_values(rng, w[n].shape, dtype if dtype != torch.float16 else torch.float32)
        tensors[n] = (t.to(torch.float16) if dtype == torch.float16 else t).cuda()
        w[n] = want
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, quant=1, quant_type=INT4)
    try:
        m.head_format(INT8)
        m.update_weights_from_tensors(tensors)
        Checker(Config(s, w, 1, INT4, head_qt=INT8)).check(m, names)
    finally:
        m.close()


TP_WORLDS = [(p, wd) for p in ("small5", "small6", "small7") for wd in (2, 4, 8)]


@pytest.mark.parametrize("preset,world", TP_WORLDS)
def test_tensor_parallel_cuts(preset, world):
    """Every rank of a world, created in turn on device 0 and never connected: each rank's fills hold its cut bit for bit, a
    split matrix holds every cell on exactly one rank and a copied matrix on every rank, the rank's vectors are its slice."""
    s = synth.PRESETS[preset]
    st = image(s)
    w = O.parse_st(st)
    holdings = {}
    for r in range(world):
        m = runtime.Model(st, max_batch=2, token_chunk_size=16, rank=r, world=world)
        try:
            ck = Checker(Config(s, w, rank=r, world=world))
            ck.check(m)
            segs = seg_tensors(s, w)
            for n in segs:
                cut = "rows" if n == "head.weight" else TP_CUTS[s.version][kind_of(n)]
                cover = ck.holdings[n]
                shape = w[n].shape
                rows, ld = (shape[1], shape[2]) if len(shape) == 3 else shape
                if cut == "rows":
                    lo, hi = r * rows // world, (r + 1) * rows // world
                    assert cover[:, lo:hi].min() == 1 and cover.sum() == cover[:, lo:hi].size, (n, r)
                elif cut == "cols":
                    lo, hi = r * ld // world, (r + 1) * ld // world
                    assert cover[:, :, lo:hi].min() == 1 and cover.sum() == cover[:, :, lo:hi].size, (n, r)
                else:
                    assert cover.min() == 1, (n, r)
                holdings[n] = holdings.get(n, 0) + cover
        finally:
            m.close()
    for n, cover in holdings.items():
        cut = "rows" if n == "head.weight" else TP_CUTS[s.version][kind_of(n)]
        assert np.all(cover == (world if cut == "copy" else 1)), (n, cut, int(cover.min()), int(cover.max()))


def test_debug_fill_refusals():
    """An unknown tensor, a fill index out of range and a buffer one byte short are ERR_INVALID, and nothing is written."""
    import ctypes as C
    st = image(synth.PRESETS["tiny6"])
    m = runtime.Model(st, max_batch=2, token_chunk_size=16)
    try:
        lib, h = capi.lib(), m._h
        assert lib.b200rwkv_debug_fills(h, b"no.such.tensor") == 0
        n = lib.b200rwkv_debug_fills(h, b"blocks.0.att.key.weight")
        assert n == 1
        info = capi.FillInfo()
        assert lib.b200rwkv_debug_fill(h, b"blocks.0.att.key.weight", 0, C.byref(info), None, 0) == capi.OK
        need = info.bytes
        assert need == 256 * 256 * 2
        out = np.full(need, 0xAB, np.uint8)
        for name, i, cap in ((b"no.such.tensor", 0, need), (b"blocks.0.att.key.weight", 1, need),
                             (b"blocks.0.att.key.weight", -1, need), (b"blocks.0.att.key.weight", 0, need - 1)):
            info.kind = 77
            assert lib.b200rwkv_debug_fill(h, name, i, C.byref(info), capi.ptr(out), cap) == capi.ERR_INVALID, (name, i, cap)
            assert info.kind == 77 and np.all(out == 0xAB), (name, i, cap)
        assert lib.b200rwkv_debug_fill(h, b"blocks.0.att.key.weight", 0, C.byref(info), capi.ptr(out), need) == capi.OK
        assert info.kind == capi.FILL_SEG and not np.all(out == 0xAB)
    finally:
        m.close()
