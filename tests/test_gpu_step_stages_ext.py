"""Every stage of real infer steps (test_gpu_step_stages.py: each stage against a float64 evaluation on the engine's own
inputs to it) on FP8 and Int4 layers and on engines whose slots are bound to unblended LoRA adapters.

Quantised layers: the first two layers FP8 or Int4, so later prefix images mix quantised and f16 layers; the reference
weight of a quantised projection is the engine contract's dequantised matrix (FP8 f32(s_n value(q)), Int4
fma_f16(q, scale, min)), in project64's bound.  The 7B-shaped layer is where the output projection and the channel-mix
value are cut into split-K slices.

Adapters (b200rwkv_create_adapters): three adapters -- rank 128 on every projection the version has, rank 5 on a subset
with the head, rank 16 on att.value alone -- at alphas 0.1 (f16(alpha lora.1) rounds), -0.37 and 2.  Every checked step
mixes slots bound to 1, 2 and 3 with unbound slots, and the binding changes between the two rounds of steps, so the
graph replays run with a new table; a last decode step with no slot bound must run the base plans.  On a step with a bound
slot, a projection some adapter pairs runs W' = [W^ | E_1 | ... | E_n], E_a = f16(alpha_a lora.1 of a) in a 128-wide
block (zeros past the rank, or for an adapter without a pair on W), on its operand [x | tail blocks], whose tails
adapter_shrink_kernel writes.  Each such projection adds two stages:
  shrink      the tail blocks read back (debug_read "<operand>_tail") against u64 = x A^T in float64 from the operand values
              the projection multiplies (hi + lo at precision 1), A = lora.0^T of the row's adapter, within
              (K/32 + 24) 2^-24 sum_k |x_k A_jk| plus half an f16 ulp (2^-22 |u| for split pairs, whose form is checked too);
              exact zeros past the rank, in every other adapter's block and in every row of an unbound slot.  The head's
              rows are its output rows.
  projection  project64 of [x | u] against [W^ | E_1 | ... | E_n]: the same GEMM over K + 128 n, so the same bound (FP8:
              the tail is not scaled by the row scale).  The residual bounds after the output projection and the
              channel-mix value gain sum_j |u_j E_nj|.
The channel mix's shrink writes the tails of the operands it multiplies, a_x0 (ffn key) and, for v5 / v6, a_x1 (ffn
receptance), so a step ends with those tails holding the channel mix's u: they are checked as that, and the time-mix
projections that multiply a_x0 / a_x1 (v5 / v6 key, v7 receptance, whose operands test_gpu_step_stages.py recomputes) take
u recomputed from the recomputed operand, its bound widened by the operand's ambiguity through |A|, and the projection's
by |E| ulp16(u) only where u lies within that bound of an f16 rounding boundary (test_gpu_step_stages.operand_rounding).
"""
import dataclasses
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

import test_gpu_step_stages as S
from test_gpu_step_stages import P

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
TAIL = 128
ALL_KINDS = ("att.receptance", "att.key", "att.value", "att.gate", "att.output", "ffn.key", "ffn.receptance", "ffn.value")
# (rank, alpha, targets, with the head)
ADAPTERS = ((128, 0.1, ALL_KINDS, True),
            (5, -0.37, ("att.key", "att.gate", "att.output", "ffn.receptance"), True),
            (16, 2.0, ("att.value",), False))


@dataclasses.dataclass(frozen=True)
class Config(S.Config):
    adapters: bool = False
    quant_adapters: bool = False


def A(name, **kw):
    return Config(P(name), adapters=True, **kw)


CONFIGS = {
    "tiny5-fp8": Config(P("tiny5"), quant="FP8"),
    "tiny6-fp8": Config(P("tiny6"), quant="FP8"),
    "tiny7-fp8": Config(P("tiny7"), quant="FP8"),
    "small6-fp8": Config(P("small6"), quant="FP8"),                  # the RWKV-6 front half feeding FP8 projections
    "tiny6-int4": Config(P("tiny6"), quant="Int4"),
    "tiny7-int4": Config(P("tiny7"), quant="Int4"),
    # production shape at V = 4096, as test_gpu_step_stages' 7b-layer: split-K slices of the quantised output projection
    # and channel-mix value
    "7b-layer-fp8": Config(P("v6-7b", L=1, V=4096), quant="FP8", batch=16, rounds=1, ragged=False),
    "7b-layer-int4": Config(P("v6-7b", L=1, V=4096), quant="Int4", batch=16, rounds=1, ragged=False),
    "tiny5-adapters": A("tiny5"),
    "tiny6-adapters": A("tiny6"),
    "tiny7-adapters": A("tiny7"),
    "small6-adapters": A("small6"),
    "small6-p1-adapters": A("small6", precision=1),                  # split tails
    "tiny6-int8-adapters": A("tiny6", quant="Int8", quant_adapters=True),
    "tiny7-nf4-adapters": A("tiny7", quant="NF4", quant_adapters=True),
    "tiny6-fp8-adapters": A("tiny6", quant="FP8", quant_adapters=True),
    "tiny7-int4-adapters": A("tiny7", quant="Int4", quant_adapters=True),
}


def adapter_files(shp):
    """The adapter files of ADAPTERS for shape `shp`, with their alphas."""
    out = []
    for i, (rank, alpha, targets, head) in enumerate(ADAPTERS):
        img = synth.make_lora_st(shp, rank=rank, seed=21 + i, targets=targets)
        if not head:
            img = synth.pack_st({k: np.asarray(v) for k, v in O.parse_st(img).items() if not k.startswith("head.")})
        out.append((img, alpha))
    return out


class AdStages(S.Stages):
    """Stages of one call on an adapter engine: `bind` [S] the adapter of every slot for this call, `loras` [(tensors,
    alpha)] of adapters 1..n."""
    bind = None
    loras = ()

    def row_ids(self, operand):
        ids = np.asarray(self.bind)[self.slot_of]
        return ids[self.out_rows] if operand == "a_head" else ids

    def pairs(self, wname):
        base = wname[:-len(".weight")]
        return [(lo.get(base + ".lora.0"), lo.get(base + ".lora.1"), alpha) for lo, alpha in self.loras]

    def proj(self, stage, x, wname, act, got, bias=None, a16=None, dz=0.0, wm=None, operand=None):
        if operand is not None and wm is None:
            pairs = self.pairs(wname)
            ids = self.row_ids(operand)
            if any(p[0] is not None for p in pairs) and ids.any():
                x, wm, dz = self.extend(operand, x, wname, pairs, ids, dz)
        return super().proj(stage, x, wname, act, got, bias, a16, dz, wm, operand)

    def extend(self, operand, x, wname, pairs, ids, dz):
        """[x | u], [W^ | E_1 | ... | E_n] and the operand error of an adapted projection on a step with a bound slot,
        after the shrink stage's checks of the tail read back (or u recomputed, when the channel mix overwrote it)."""
        n, (R, K) = len(pairs), x.shape
        Wm = self.mat(wname)
        E = np.zeros((Wm.shape[0], TAIL * n))
        own = np.zeros((R, TAIL * n), bool)                     # (row, column) where the row's u lives
        ref, acc = np.zeros((R, TAIL * n)), np.zeros((R, TAIL * n))
        recomputed = wname in self.recomputed
        if recomputed:                                            # the operand as the kernel must have rounded it
            xv, ex = S.operand_rounding(*self.recomputed[wname], self.split)
        else:
            xv, ex = x, 0.0
        for a, (l0, l1, alpha) in enumerate(pairs):
            if l0 is None:
                continue
            r = l0.shape[1]
            E[:, a * TAIL:a * TAIL + r] = (np.float32(alpha) * np.asarray(l1, np.float32)).astype(np.float16)
            rows = ids == a + 1
            if not rows.any():
                continue
            Am = np.asarray(l0, np.float64)                       # lora.0 = A^T [K, r]
            cols = slice(a * TAIL, a * TAIL + r)
            own[np.ix_(rows, np.arange(a * TAIL, a * TAIL + r))] = True
            ref[rows, cols] = xv[rows] @ Am
            acc[rows, cols] = (K / 32 + 24) * EPS * (np.abs(xv[rows]) @ np.abs(Am))
            if recomputed:
                acc[rows, cols] += (ex[rows] if np.ndim(ex) else ex) @ np.abs(Am)
        short = wname.split(".", 2)[-1] if wname.startswith("blocks.") else wname
        if recomputed:
            # the tail holds the channel mix's u by now: u as the shrink must have rounded it, the ambiguity through |E|
            u, eu = S.operand_rounding(ref, acc, self.split)
            u, eu = np.where(own, u, 0.0), np.where(own, eu, 0.0)
            dz = dz + eu @ np.abs(E).T
        else:
            bits, u = self.rd.a16(operand + "_tail", TAIL * n, R)
            if self.split:
                bound = acc + 2.0 ** -22 * np.abs(ref) + 2.0 ** -40
            else:
                bound = acc + S.LN.f16_ulp(ref) / 2 + 2.0 ** -25
            self.ck(f"shrink u {short} ({operand}_tail)", u, ref, np.where(own, bound, np.inf))
            zero = np.concatenate([bits[:R][~own]] + ([bits[16:16 + R][~own]] if self.split else []))
            self.ck.exact(f"shrink zeros {short} ({operand}_tail)", zero.astype(np.float32), np.zeros(zero.shape, np.float32))
        self.tail_sum[wname] = np.abs(u) @ np.abs(E).T
        return np.concatenate([x, u], 1), np.concatenate([Wm.astype(np.float64), E], 1), dz


class AdRunner(S.Runner):
    stages = AdStages

    def plan(self):
        """test_gpu_step_stages' plan with a fourth entry in the 17..128-token step (so that it too holds slots of all three
        adapters and an unbound one), then a decode step with no slot bound."""
        plan = S.step_plan(self.cfg)
        rng = np.random.default_rng(zlib.crc32(repr(self.cfg).encode()) + 1)
        self.perm = [e[0] for e in dict(plan)["decode0"]]
        out = []
        for tag, ent in plan:
            if tag.startswith("prompt"):
                ent = ent + [(self.perm[1], 7, S.FULL, rng.integers(0, self.cfg.shape.V, 7).tolist())]
            out.append((tag, ent))
        return out + [("unbound", dict(plan)["decode0"])]

    def binding(self, tag):
        """Adapter of every slot: the slots perm[0..3] of the ragged and 17..128-token steps hold adapters 1, 2, 3 and
        none in both rounds, in another order in round 1."""
        ids = np.zeros(self.cfg.batch, np.int32)
        if tag == "unbound":
            return ids
        order = (1, 2, 3, 0, 2, 0, 1, 3) if tag == "warmup" or tag.endswith("0") else (3, 0, 1, 2, 0, 1, 3, 2)
        for i, s in enumerate(self.perm):
            ids[s] = order[i % len(order)]
        return ids

    def model_kw(self, shp):
        kw = super().model_kw(shp)
        files = adapter_files(shp)
        self.loras = [(dict(O.parse_st(img)), alpha) for img, alpha in files]
        return dict(kw, adapters=files, quant_adapters=self.cfg.quant_adapters)

    def before(self, m, tag, sg=None):
        ids = self.binding(tag)
        if sg is None:
            m.bind_adapter(list(range(self.cfg.batch)), ids.tolist())
        else:
            sg.bind, sg.loras = ids, self.loras


@pytest.mark.parametrize("name", list(CONFIGS))
def test_step_stages(name):
    cfg = CONFIGS[name]
    (AdRunner if cfg.adapters else S.Runner)(name, cfg).run()


def test_tail_read_needs_adapters():
    """`<operand>_tail` reads the n_adapters x 128 tail columns of a projection operand; an engine without adapters, or an
    operand without tails, refuses it, and the plain names keep their widths."""
    st = synth.make_st("tiny6", 0)
    m = runtime.Model(st, max_batch=4, token_chunk_size=128)
    try:
        m.infer_raw([0, 1], [2, 1], [5, 7, 9], [S.LAST, S.LAST])
        for name in ("a_x2_tail", "a_head_tail", "a_kk_tail_lo"):
            with pytest.raises(capi.B200Error) as e:
                m.debug_read(name, 3)
            assert e.value.code == capi.ERR_STATE
    finally:
        m.close()
    files = adapter_files(synth.PRESETS["tiny6"])
    m = runtime.Model(st, max_batch=4, token_chunk_size=128, adapters=files)
    try:
        m.bind_adapter([0, 1], [1, 0])
        m.infer_raw([0, 1], [2, 1], [5, 7, 9], [S.LAST, S.LAST])
        assert m.debug_read("a_x2", 3).shape == (3, 256)
        assert m.debug_read("a_kk", 3).shape == (3, 896)
        tail = m.debug_read("a_x2_tail", 3)
        assert tail.shape == (3, TAIL * len(files))
        assert tail[:2, :128].any() and not tail[:2, 128:].any() and not tail[2].any()
        with pytest.raises(capi.B200Error) as e:
            m.debug_read("a_lora0_0_tail", 3)
        assert e.value.code == capi.ERR_STATE
        with pytest.raises(capi.B200Error) as e:
            m.debug_read("a_x2_tail_lo", 3)
        assert e.value.code == capi.ERR_STATE
    finally:
        m.close()
