"""Every stage of the last layer of real infer steps, each held to a float64 evaluation of that stage on the engine's own
inputs to it, read back with b200rwkv_debug_read.

The kernel tests (test_gpu_gemm.py, test_gpu_ln.py, test_gpu_wkv.py) hold each kernel to a float64 reference on inputs
they build.  What they cannot see is the step program the engine builds at load: which buffer feeds which projection,
which weight and which layer's vectors each launch takes, which activation and output form (f32 rows, an f16 operand, a
split hi + lo pair) each segment gets, how the split-K slices and gates reach the next LN stage, and which rows the
token-shift commits copy.  Logits and states tolerate many such errors (a projection output rounded to f16 moves the
logits by less than 1e-3; a lost lo half at precision 1 by 2e-6 to 1e-4), so this file checks every stage alone.

Each stage takes the engine's own output of the stage before it (read back), so each bound is that stage's own rounding
bound, with the kernel tests' formulas (test_gpu_gemm.project64, test_gpu_ln.ln_ref / residual_ref / f16_got,
test_gpu_wkv.reference / decay_of):
  LN1        x_a: LN0 of the embedding row at layer 0; at layer l > 0 the previous prefix model's `hidden` row (two
             residual bounds); xx1 = LN1(x_a); sx1 = prev - xx1 (prev: the slot's att shift before the call for an entry's
             first token, else the previous token's xx1; only RWKV-6 writes sx1, v5 / v7 mix from it inside the LN
             kernel); the mixes (v5 1 - mu, v6 time_mix_x and the ddlerp LoRA, v7 six lerps);
  projections r / k / v / g, the decay / a / v / g LoRA stages, the output projection (split-K slices summed), channel-mix
             key (relu^2) and receptance (sigmoid), channel-mix value, head: each output against W (the operand read back),
             W the f16 or dequantised weight;
  WKV        a_out and the slot states after the call against the recurrence from the r / k / v / g / w / a / nu /
             v_first rows read back and the states before the call; with the RWKV-6 decay fold, w is never written and
             comes from a_lora1 and time_decay_w2 (decay_of);
  LN2        x_b = x_a + att; xx2 = LN2(x_b); the channel-mix mixes;
  ln_out     hidden = x_b + rr (.) ffn (v7: + ffn); the a_head rows of the tokens with logits rows = ln_out(hidden); the
             logits infer returned = a_head head^T;
  commits    bit for bit: the slot's att shift equals the xx1 row of the entry's last token, its ffn shift that token's
             xx2 row.
Operands the channel-mix LN overwrites (v5 the k mix, v6 the decay-LoRA input and the k mix, v7 the r mix) are recomputed
from xx1, sx1 and the mix vectors; the projection bound then widens by sum_k |W_nk| ulp16(x_k) only where the recomputed
value lies within its own error bound of an f16 rounding boundary (with split operands, by |W| times the pair's error).

The buffers hold the last layer of the last step, so a model of L layers runs as its prefix images blocks.0..l + ln_out +
head for l = 0 .. L - 1: each layer is the last layer once.  Each image runs the same calls: a warm-up prompt in every
slot (not checked), then a decode batch, a ragged step of <= 16 tokens and a 17..128-token step of three entries (LAST /
FULL / NONE), twice in that order, so that graph replays are checked as well as first captures (the two production
shapes: the decode batch and the 40-token step once, then the decode batch again).  Precision 1 runs every step at
<= 16 tokens, so it has no 17..128-token step.

Every split (hi + lo) operand read back at precision 1 is also checked for its form, independent of any GEMM bound: hi
is a nearest f16 of hi + lo and lo is nonzero for most elements, so a stage that writes a plain f16 operand where a split
one is due fails even when the rounding it costs stays inside the consumer's bound.
"""
import dataclasses
import types
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

import fp8_oracle as F8
import int4_oracle as I4
import test_gpu_gemm as G
import test_gpu_ln as LN
import test_gpu_wkv as W

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
LAST, FULL, NONE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE


@dataclasses.dataclass(frozen=True)
class Config:
    shape: synth.Shape
    precision: int = 0
    quant: str = ""
    batch: int = 8
    rounds: int = 2                 # times the step shapes run (the second round replays the step graphs)
    ragged: bool = True             # the step of <= 16 tokens from several tokens per slot


def P(name, **over):
    return dataclasses.replace(synth.PRESETS[name], **over)


CONFIGS = {
    "tiny5": Config(P("tiny5")),
    "tiny6": Config(P("tiny6")),
    "tiny7": Config(P("tiny7")),
    "small6": Config(P("small6")),                                   # RWKV-6 front half, decay fold
    "small7": Config(P("small7")),
    "small6-Dd192": Config(P("small6", Dd=192)),                    # decay LoRA stage 2 as its own launch
    "small6-Dm16": Config(P("small6", Dm=16)),                      # no front half: LN1 + W1 + W2
    "small6-Dm64": Config(P("small6", Dm=64)),
    "small6-C320": Config(P("small6", C=320, F=1152)),              # C not a multiple of 128
    "small7-2b9ranks": Config(P("small7", Dd=96, Da=96, Dv=64, Dg=320)),
    "tiny5-p1": Config(P("tiny5"), precision=1),
    "small6-p1": Config(P("small6"), precision=1),
    "tiny7-p1": Config(P("tiny7"), precision=1),
    "tiny6-int8": Config(P("tiny6"), quant="Int8"),
    "tiny7-int8": Config(P("tiny7"), quant="Int8"),
    "tiny6-nf4": Config(P("tiny6"), quant="NF4"),
    "tiny7-nf4": Config(P("tiny7"), quant="NF4"),
    # production shapes at V = 4096: split-K slices > 1 on the output projection and the channel-mix value.  Their float64
    # references dominate the file's run time, so they run the decode batch and the 40-token step, then the decode graph once
    # more as a replay.
    "7b-layer": Config(P("v6-7b", L=1, V=4096), batch=16, rounds=1, ragged=False),
    "2b9-2layers": Config(P("v7-2b9", L=2, V=4096), rounds=1, ragged=False),
}
QUANT_LAYERS = 2


def step_plan(cfg: Config):
    """The calls of one image: (tag, entries [(slot, tokens, option, token ids)]).  Tokens come from a generator seeded by
    the config, so every prefix image gets the same inputs.  The first call, "warmup", only makes the states non-zero."""
    B = cfg.batch
    rng = np.random.default_rng(zlib.crc32(repr(cfg).encode()))
    perm = [int(s) for s in rng.permutation(B)]
    dec = [(s, 1, LAST) for s in perm]
    rag = [(perm[1], 5, FULL), (perm[0], 1, LAST), (perm[3], 6, NONE), (perm[2], 3, LAST)]
    big = [(perm[2], 23, LAST), (perm[0], 9, FULL), (perm[3], 8, NONE)]
    shapes = [("decode", dec)] + ([("ragged", rag)] if cfg.ragged else []) + ([("prompt", big)] if cfg.precision == 0 else [])
    plan = [("warmup", [(s, 3 if cfg.precision == 0 else 2, NONE) for s in range(B)])]
    for rnd in range(cfg.rounds):
        plan += [(f"{tag}{rnd}", ent) for tag, ent in shapes]
    if cfg.rounds == 1:
        plan.append(("decode1", dec))
    V = cfg.shape.V
    return [(tag, [(s, n, o, rng.integers(0, V, n).tolist()) for s, n, o in ent]) for tag, ent in plan]


# ---- reading the engine back ------------------------------------------------------------------------------------------
class Reader:
    def __init__(self, m, T, split, ck):
        self.m, self.T, self.split, self.ck = m, T, split, ck

    def f32(self, name):
        return self.m.debug_read(name, self.T).astype(np.float64)

    def a16(self, name, K, n=None):
        """(bits [rows, K] in the A16 token-row order of test_gpu_ln.f16_got, value hi (+ lo) [n, K] f64) of the first n
        rows (default: every token of the step)."""
        T = self.T if n is None else n
        hi = self.m.debug_read(name, self.T)[:T, :K]
        bits = np.zeros((32 if self.split else T, K), np.uint16)
        bits[:T] = hi.astype(np.float16).view(np.uint16)
        val = hi.astype(np.float64)
        if self.split:
            lo = self.m.debug_read(name + "_lo", self.T)[:T, :K]
            self.ck.pair(name, hi, lo)
            bits[16:16 + T] = lo.astype(np.float16).view(np.uint16)
            val = val + lo.astype(np.float64)
        return bits, val


class Checker:
    """Worst error / bound per stage; every stage over 1 is reported with its worst token and column."""

    def __init__(self, tag):
        self.tag, self.worst, self.bad = tag, {}, []

    def __call__(self, stage, got, want, bound):
        err = np.abs(np.asarray(got, np.float64) - want)
        r = np.where(np.isnan(err), np.inf, err / bound)
        w = float(np.max(r, initial=0.0))
        self.worst[stage] = max(self.worst.get(stage, 0.0), w)
        if w > 1.0:
            i = np.unravel_index(int(np.argmax(r)), r.shape)
            self.bad.append(f"{stage}: error / bound {w:.3g} at (token, column) {tuple(int(v) for v in i)}: "
                            f"got {np.broadcast_to(got, r.shape)[i]!r}, want {np.broadcast_to(want, r.shape)[i]!r}")

    def pair(self, name, hi, lo):
        """A split operand read back, whatever its stage's bound: hi is a nearest f16 of hi + lo (lo at most half the f16
        spacing on its side of hi; pairs saturated at 65504 excepted), and lo carries the rest of the f32 value, so it is
        nonzero for most elements.  A lo half lost on the way (a plain f16 operand, lo rows left zero) fails here even
        where the rounding it costs stays inside the stage's bound."""
        h = np.asarray(hi, np.float16)
        a = np.abs(h)
        with np.errstate(over="ignore"):          # the step above 65504 is inf; those pairs are excepted below
            up = (np.nextafter(a, np.float16(np.inf)) - a).astype(np.float64)
        dn = np.where(a == 0, up, (a - np.nextafter(a, np.float16(0))).astype(np.float64))
        sl = np.asarray(lo, np.float64) * np.where(h < 0, -1.0, 1.0)
        sat = a == np.float16(LN.F16_MAX)
        near = sat | ((sl <= up / 2) & (sl >= -dn / 2))
        live = (h != 0) & ~sat
        n = int(np.count_nonzero(live))
        carried = np.count_nonzero(np.asarray(lo)[live] != 0) / max(n, 1)
        stage = f"split pair {name}"
        self.worst[stage] = max(self.worst.get(stage, 0.0), 0.0 if near.all() and (n < 16 or carried >= 0.5) else np.inf)
        if not near.all():
            i = tuple(int(v) for v in np.argwhere(~near)[0])
            self.bad.append(f"{stage}: hi is not the nearest f16 of hi + lo at (token, column) {i}: hi {h[i]!r}, lo {lo[i]!r}")
        if n >= 16 and carried < 0.5:
            self.bad.append(f"{stage}: lo is zero for {1 - carried:.0%} of the nonzero elements: the lo half was lost")

    def exact(self, stage, got, want):
        ok = np.array_equal(np.ascontiguousarray(got, np.float32).view(np.uint32), np.ascontiguousarray(want, np.float32).view(np.uint32))
        self.worst[stage] = 0.0 if ok else np.inf
        if not ok:
            self.bad.append(f"{stage}: not bit-identical")

    def done(self):
        print(f"\n[stages] {self.tag}: " + " ".join(f"{k} {v:.3f}" for k, v in self.worst.items()))
        assert not self.bad, f"{self.tag}: " + "; ".join(self.bad)


# ---- per-stage references -----------------------------------------------------------------------------------------------
def mix_ref(xx, sx, mu, dsx=0.0):
    """y = xx + sx mu from the kernel's own xx and sx (dsx: error of sx when it is recomputed here)."""
    y = xx + sx * mu
    return y, np.abs(mu) * dsx + 2 * EPS * (np.abs(sx * mu) + np.abs(y))


def operand_rounding(y, dy, split):
    """A value y (error bound dy) the kernel stored as an operand that could not be read back: the value as the kernel must
    have rounded it, and the error e_k it may still carry (with split operands the pair's error, else one f16 ulp only where
    y lies within dy of an f16 rounding boundary)."""
    if split:
        return y, dy + 2.0 ** -22 * np.abs(y) + 2.0 ** -25
    c = lambda v: np.clip(v, -LN.F16_MAX, LN.F16_MAX).astype(np.float16).astype(np.float64)
    amb = c(y - dy) != c(y + dy)                     # within its bound of an f16 rounding boundary
    return c(y), np.where(amb, LN.f16_ulp(y), 0.0)


def recomputed_operand(y, dy, split, Wm):
    """An operand that was overwritten before it could be read back: its value as the kernel must have rounded it, and
    the projection error that the rounding ambiguity can add, sum_k |W_nk| e_k."""
    x, e = operand_rounding(y, dy, split)
    return x, (e @ np.abs(Wm.astype(np.float64)).T if e.any() else 0.0)


class Stages:
    """The checks of one infer call of one prefix image (its last layer l)."""

    def __init__(self, cfg: Config, wts, l, entries, rd: Reader, ck: Checker, st0, st1):
        self.cfg, self.s, self.w, self.l = cfg, cfg.shape, wts, l
        self.rd, self.ck, self.split = rd, ck, cfg.precision == 1
        self.entries, self.st0, self.st1 = entries, st0, st1
        self.first, self.last, self.slot_of = [], [], []
        for s, n, _, _ in entries:
            self.first += [True] + [False] * (n - 1)
            self.last += [False] * (n - 1) + [True]
            self.slot_of += [s] * n
        self.first, self.last, self.slot_of = np.array(self.first), np.array(self.last), np.array(self.slot_of)
        self.T = len(self.slot_of)
        self.out_rows = None           # the tokens with logits rows, once ln_out is checked
        self.recomputed = {}           # projection weight -> (value, bound) of its recomputed operand (recomputed_op)
        self.tail_sum = {}             # projection weight -> sum |x_k W_nk| over columns beyond its own (Stages.residual)

    def mat(self, name):
        return self.w[name]

    def vec(self, name):
        return np.asarray(self.w[name], np.float32).reshape(-1).astype(np.float64)

    def prev_rows(self, own, state_row):
        """prev of every token: the slot's shift row from before the call for an entry's first token, else the previous
        token's row of `own`."""
        before = self.st0[self.slot_of, self.l, state_row].astype(np.float64)
        return np.where(self.first[:, None], before, np.roll(own, 1, 0))

    def recomputed_op(self, y, dy, wname):
        """recomputed_operand for the projection `wname`, whose operand the channel mix overwrote."""
        self.recomputed[wname] = (y, dy)
        return recomputed_operand(y, dy, self.split, self.mat(wname))

    def proj(self, stage, x, wname, act, got, bias=None, a16=None, dz=0.0, wm=None, operand=None):
        """One projection against float64; `operand`: the A16 buffer the engine multiplies (a projection an adapter can
        extend, test_gpu_step_stages_ext.py)."""
        Wm = self.mat(wname) if wm is None else wm
        y, b = G.project64(x, Wm, bias, act, G.EPS, dz)
        if a16 is None:
            self.ck(stage, got, y, b)
        else:
            g, want, bound = LN.f16_got(a16, y, b, self.split, self.T)
            self.ck(stage, g, want, bound)
        return y, b

    def op(self, name, K):
        return self.rd.a16(name, K)

    def run(self, x_a_want):
        s, l, T, split, ck = self.s, self.l, self.T, self.split, self.ck
        C, N, H = s.C, s.N, s.H
        b, a, f = f"blocks.{l}.", f"blocks.{l}.att.", f"blocks.{l}.ffn."
        cluster = T <= 16
        rd = self.rd
        x_a, xx1, sx1 = rd.f32("x_a"), rd.f32("xx1"), rd.f32("sx1")
        # ---- LN1 ----
        if l == 0:
            tok = np.concatenate([t for _, _, _, t in self.entries])
            y, dy = LN.ln_ref(np.asarray(self.w["emb.weight"][tok], np.float32), self.vec("blocks.0.ln0.weight"),
                              self.vec("blocks.0.ln0.bias"), C, False)
            ck("LN0 x_a", x_a, y, dy)
        else:
            want, bound = x_a_want
            ck("LN1 x_a (previous image's hidden)", x_a, want, bound)
        y, dy = LN.ln_ref(x_a, self.vec(b + "ln1.weight"), self.vec(b + "ln1.bias"), C, cluster)
        ck("LN1 xx1", xx1, y, dy)
        sx = self.prev_rows(xx1, 0) - xx1
        ver = s.version
        dsx1 = 0.0
        if ver == 6:
            ck("LN1 sx1", sx1, sx, EPS * np.abs(sx) + 1e-300)
        else:                          # v5 / v7 mix inside the LN kernel and do not write sx1
            sx1, dsx1 = sx, EPS * np.abs(sx)
        ops = {}                       # projection operands: value [T, K] and the error they may carry (dz)

        def static_mix(stage, i, mu, overwritten=False, wname=None):
            y, dy = mix_ref(xx1, sx1, mu, dsx1)
            if overwritten:
                ops[i] = self.recomputed_op(y, dy, wname)
            else:
                bits, val = self.op(f"a_x{i}", C)
                g, want, bound = LN.f16_got(bits, y, dy, split, T)
                ck(stage, g, want, bound)
                ops[i] = (val, 0.0)

        if ver == 5:
            one_minus = lambda n: (np.float32(1) - np.asarray(self.w[a + n], np.float32).reshape(-1)).astype(np.float64)
            static_mix("LN1 mix k (1 - mu)", 1, one_minus("time_mix_k"), overwritten=True, wname=a + "key.weight")
            static_mix("LN1 mix v (1 - mu)", 2, one_minus("time_mix_v"))
            static_mix("LN1 mix r (1 - mu)", 3, one_minus("time_mix_r"))
            static_mix("LN1 mix g (1 - mu)", 4, one_minus("time_mix_g"))
        elif ver == 6:
            Dm = s.Dm
            static_mix("LN1 mix x (time_mix_x)", 5, self.vec(a + "time_mix_x"))
            W1 = self.mat(a + "time_mix_w1")
            W2 = self.mat(a + "time_mix_w2")
            names = ("time_mix_w", "time_mix_k", "time_mix_v", "time_mix_r", "time_mix_g")
            for j in range(5):
                bits, lora = self.op(f"a_lora0_{j}", Dm)
                self.proj(f"ddlerp W1 group {j}", ops[5][0], None, capi.ACT_TANH, None, a16=bits, wm=W1[j * Dm:(j + 1) * Dm])
                yl, dyl = G.project64(lora, W2[j], None, capi.ACT_NONE, G.EPS)
                mu = self.vec(a + names[j])
                y = xx1 + sx1 * (mu + yl)
                dy = np.abs(sx1) * dyl + 2.0 ** -22 * (np.abs(xx1) + np.abs(sx1) * (np.abs(mu) + np.abs(yl)))
                if j <= 1:             # the decay-LoRA input and the k mix: overwritten by the channel-mix LN
                    ops[j] = self.recomputed_op(y, dy, a + ("time_decay_w1" if j == 0 else "key.weight"))
                else:
                    bits, val = self.op(f"a_x{j}", C)
                    g, want, bound = LN.f16_got(bits, y, dy, split, T)
                    ck(f"ddlerp W2 mix {names[j]}", g, want, bound)
                    ops[j] = (val, 0.0)
        else:
            names = ("x_r", "x_w", "x_k", "x_v", "x_a", "x_g")
            for i, n in enumerate(names):
                static_mix(f"LN1 mix {n}", i, self.vec(a + n), overwritten=(i == 0), wname=a + "receptance.weight")
        # ---- projections in front of WKV ----
        rows = {}
        if ver in (5, 6):
            rk = dict(r=3, k=1, v=2, g=4)
        else:
            rk = dict(r=0, k=2, v=3)
        wn = dict(r="receptance", k="key", v="value", g="gate")
        for n, i in rk.items():
            rows[n] = rd.f32(n)
            x, dz = ops[i]
            self.proj(f"att {wn[n]} (a_x{i})", x, a + wn[n] + ".weight", capi.ACT_SILU if n == "g" else capi.ACT_NONE, rows[n], dz=dz,
                      operand=f"a_x{i}")
        Dd = s.Dd
        wk = W.Case(version=ver, entries=tuple((sl, n) for sl, n, _, _ in self.entries), H=H, precision=self.cfg.precision)
        ch = dict(lnx_w=np.float32(self.vec(a + "ln_x.weight")), lnx_b=np.float32(self.vec(a + "ln_x.bias")))
        tok = {n: np.float32(rows[n]) for n in rows}
        if ver == 6:
            bits, d1 = self.op("a_lora1_0", Dd)
            x, dz = ops[0]
            self.proj("decay LoRA stage 1 (tanh)", x, a + "time_decay_w1", capi.ACT_TANH, None, a16=bits, dz=dz)
            td = self.vec(a + "time_decay")
            if Dd <= 128 and Dd % 8 == 0:          # folded into the WKV kernel: w comes from d1
                wk = dataclasses.replace(wk, Dd=Dd)
                tok["d1"] = np.float32(d1)
                ch["time_decay_w2"] = np.asarray(self.w[a + "time_decay_w2"], np.float32).astype(np.float16)
                ch["decay_bias"] = np.float32(td)
            else:
                rows["w"] = rd.f32("w")
                self.proj("decay LoRA stage 2 (exp -exp)", d1, a + "time_decay_w2", capi.ACT_EXPNEGEXP, rows["w"], bias=td)
                tok["w"] = np.float32(rows["w"])
            ch["u"] = np.float32(self.vec(a + "time_first"))
        elif ver == 5:
            ch["u"] = np.float32(self.vec(a + "time_first"))
            ch["w"] = np.exp(-np.exp(self.vec(a + "time_decay")))
        else:
            lora = {}
            for j, (n1, D, x_i, act1) in enumerate((("w1", s.Dd, 1, capi.ACT_TANH), ("a1", s.Da, 4, capi.ACT_NONE),
                                                     ("v1", s.Dv, 3, capi.ACT_NONE), ("g1", s.Dg, 5, capi.ACT_SIGMOID))):
                if n1 == "v1" and l == 0:
                    continue
                bits, lora[n1] = self.op(f"a_lora{j}_0", D)
                self.proj(f"LoRA {n1}", ops[x_i][0], a + n1, act1, None, a16=bits, dz=ops[x_i][1])
            stage2 = [("w2", "w1", "w", capi.ACT_V7DECAY, "w0"), ("a2", "a1", "a", capi.ACT_SIGMOID, "a0"),
                      ("g2", "g1", "g", capi.ACT_NONE, None)]
            if l > 0:
                stage2.append(("v2", "v1", "nu", capi.ACT_SIGMOID, "v0"))
            for n2, n1, out, act, bias in stage2:
                rows[out] = rd.f32(out)
                self.proj(f"LoRA {n2} -> {out}", lora[n1], a + n2, act, rows[out], bias=None if bias is None else self.vec(a + bias))
                tok[out] = np.float32(rows[out])
            for n in ("k_k", "k_a", "r_k"):
                ch[n] = np.float32(self.vec(a + n))
            vf = rd.f32("v_first")
            if l == 0:
                ck.exact("v_first = layer 0's v", vf, rows["v"])
            else:
                ck.exact("v_first = image 0's v", vf, self.v_first0)
                tok["v_first"] = np.float32(vf)
            self.v_first = rows["v"] if l == 0 else None
        # ---- WKV ----
        M0 = {}
        for sl, _, _, _ in self.entries:
            M0[sl] = self.wkv_state(self.st0, sl)
        y, dy, states = W.reference(wk, ch, tok, M0, l)
        bits, a_out = self.op("a_out", C)
        g, want, bound = LN.f16_got(bits, y, dy, split, T)
        ck("WKV a_out", g, want, bound)
        for sl, (M, E) in states.items():
            ck("WKV state", self.wkv_state(self.st1, sl), M, E + EPS * np.abs(M) + 1e-30)
        # ---- output projection, LN2 ----
        part_att = rd.f32("part_att")
        self.proj("output projection (slices summed)", a_out, a + "output.weight", capi.ACT_NONE, part_att, operand="a_out")
        x_b = rd.f32("x_b")
        want, bound = self.residual(x_a, part_att, None, a_out, a + "output.weight", G.pick_split(C, -(-C // 128)))
        ck("LN2 x_b = x_a + att", x_b, want, bound)
        xx2 = rd.f32("xx2")
        y, dy = LN.ln_ref(x_b, self.vec(b + "ln2.weight"), self.vec(b + "ln2.bias"), C, cluster)
        ck("LN2 xx2", xx2, y, dy)
        sx2 = self.prev_rows(xx2, N + 1) - xx2
        if ver == 7:
            fm = [("x_k", 0, self.vec(f + "x_k"))]
        elif ver == 6:
            fm = [("time_mix_k", 0, self.vec(f + "time_mix_k")), ("time_mix_r", 1, self.vec(f + "time_mix_r"))]
        else:
            om = lambda n: (np.float32(1) - np.asarray(self.w[f + n], np.float32).reshape(-1)).astype(np.float64)
            fm = [("time_mix_k (1 - mu)", 0, om("time_mix_k")), ("time_mix_r (1 - mu)", 1, om("time_mix_r"))]
        fops = {}
        for n, i, mu in fm:
            y, dy = mix_ref(xx2, sx2, mu, EPS * np.abs(sx2))
            bits, val = self.op(f"a_x{i}", C)
            g, want, bound = LN.f16_got(bits, y, dy, split, T)
            ck(f"LN2 mix {n}", g, want, bound)
            fops[i] = val
        # ---- channel mix ----
        F = s.F
        bits, kk = self.op("a_kk", F)
        self.proj("ffn key (relu^2)", fops[0], f + "key.weight", capi.ACT_RELU2, None, a16=bits, operand="a_x0")
        rr = None
        if ver != 7:
            rr = rd.f32("rr")
            self.proj("ffn receptance (sigmoid)", fops[1], f + "receptance.weight", capi.ACT_SIGMOID, rr, operand="a_x1")
        part_ffn = rd.f32("part_ffn")
        self.proj("ffn value (slices summed)", kk, f + "value.weight", capi.ACT_NONE, part_ffn, operand="a_kk")
        hidden = rd.f32("hidden")
        hid_want, hid_bound = self.residual(x_b, part_ffn, rr, kk, f + "value.weight", G.pick_split(F, -(-C // 128)))
        ck("ln_out hidden = x_b + ffn", hidden, hid_want, hid_bound)
        # ---- ln_out, head, logits ----
        outrow = []
        for _, n, o, _ in self.entries:
            outrow += [o == FULL or (o == LAST and j == n - 1) for j in range(n)]
        toks = np.nonzero(outrow)[0]
        R = len(toks)
        self.out_rows = toks
        if R:
            y, dy = LN.ln_ref(hidden[toks], self.vec("ln_out.weight"), self.vec("ln_out.bias"), C, False)
            bits, head_in = rd.a16("a_head", C, R)
            g, want, bound = LN.f16_got(bits, y, dy, split, R)
            ck("ln_out a_head", g, want, bound)
            self.proj("head logits", head_in, "head.weight", capi.ACT_NONE, self.logits, operand="a_head")
        # ---- commits ----
        last = np.nonzero(self.last)[0]
        slots = self.slot_of[last]
        ck.exact("commit att shift = xx1 of the last token", self.st1[slots, l, 0], xx1[last])
        ck.exact("commit ffn shift = xx2 of the last token", self.st1[slots, l, N + 1], xx2[last])
        return x_a, hidden, 2 * hid_bound

    def residual(self, x, part, gate, op, wname, nsplit):
        """x + gate (.) part, with part the split-K slices summed (by the kernel, and by debug_read in slice order): the
        bound of test_gpu_ln.residual_ref with sum |slice| <= sum_k |op_k W_nk| (over the operand's own columns and any
        tail columns the projection multiplied), plus the f32 sum of the slices."""
        c = types.SimpleNamespace(n_parts=1, n_gate=1 if gate is not None else 0)
        xs = dict(x_in=[x], parts=[part[None]], gates=[gate[None]] if gate is not None else None)
        y, dy = LN.residual_ref(c, xs, 0)
        sa = np.abs(op) @ np.abs(self.mat(wname).astype(np.float64)).T + self.tail_sum.get(wname, 0.0)
        g = np.abs(gate) if gate is not None else 1.0
        return y, dy + 2 * EPS * (nsplit + 2) * g * sa + 1e-300

    def wkv_state(self, st, slot):
        N, H = self.s.N, self.s.H
        S = st[slot, self.l, 1:1 + N].astype(np.float64).reshape(N, H, N).transpose(1, 0, 2)     # S[h][row][col]
        return S if self.s.version == 7 else S.transpose(0, 2, 1)                                 # M[h][value][key]


def weights_of(st, cfg: Config):
    """The model's weights as the engine multiplies them: the first QUANT_LAYERS layers' projection matrices dequantised by
    the format's engine contract (FP8: f32(s_n value(q)); Int4: fma_f16(q, scale, min))."""
    w = dict(O.parse_st(st))
    if cfg.quant:
        qt = {"Int8": Q.QUANT_INT8, "NF4": Q.QUANT_NF4, "FP8": F8.QUANT_FP8, "Int4": I4.QUANT_INT4}[cfg.quant]
        w = (I4 if qt == I4.QUANT_INT4 else F8).quantize_model(w, QUANT_LAYERS, qt)
    return {k: (v if k == "emb.weight" else np.asarray(v, np.float32)) for k, v in w.items()}


class Runner:
    """The prefix images of one config and the plan's calls on each, every call but the warm-up checked stage by stage.
    test_gpu_step_stages_ext.py extends the engine (`model_kw`), binds slots before each call (`before`) and checks with
    its own `stages`."""
    stages = Stages

    def __init__(self, name, cfg: Config):
        self.name, self.cfg = name, cfg

    def plan(self):
        return step_plan(self.cfg)

    def model_kw(self, shp):
        return dict(quant=QUANT_LAYERS, quant_type=self.cfg.quant) if self.cfg.quant else {}

    def before(self, m, tag, sg=None):
        """Before the call `tag` (sg None), and before its checks (sg: the call's Stages)."""

    def run(self):
        cfg = self.cfg
        s = cfg.shape
        plan = self.plan()
        prev = {}                      # step tag -> (hidden, bound) of the previous prefix image
        v0 = {}                        # step tag -> layer 0's v rows (v7)
        for l in range(s.L):
            shp = dataclasses.replace(s, L=l + 1)
            st = synth.make_st(shp, 0)
            wts = weights_of(st, cfg)
            m = runtime.Model(st, max_batch=cfg.batch, token_chunk_size=128, exact=cfg.precision == 1, **self.model_kw(shp))
            try:
                cur = {}
                for tag, entries in plan:
                    slots = [e[0] for e in entries]
                    self.before(m, tag)
                    st0 = np.stack([m.state.back(b) for b in range(cfg.batch)])
                    out = m.infer_raw(slots, [e[1] for e in entries], sum((e[3] for e in entries), []), [e[2] for e in entries])
                    st1 = np.stack([m.state.back(b) for b in range(cfg.batch)])
                    T = sum(e[1] for e in entries)
                    if tag == "warmup":
                        continue
                    ck = Checker(f"{self.name} layer {l} {tag} T={T}")
                    sg = self.stages(cfg, wts, l, entries, Reader(m, T, cfg.precision == 1, ck), ck, st0, st1)
                    sg.logits = np.concatenate([r for r in out if len(r)]) if any(len(r) for r in out) else None
                    sg.v_first0 = v0.get(tag)
                    self.before(m, tag, sg)
                    _, hidden, hb = sg.run(prev.get(tag))
                    cur[tag] = (hidden, hb)
                    if l == 0 and s.version == 7:
                        v0[tag] = sg.v_first
                    ck.done()
                prev = cur
            finally:
                m.close()


def run_config(name):
    Runner(name, CONFIGS[name]).run()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_step_stages(name):
    run_config(name)


def test_lo_half_needs_split_operands():
    """`<operand>_lo` reads the lo halves of split operands; after a step without them it is refused, and the hi halves of
    a split step are the f16 rounding of the value with the lo halves the rest."""
    st = synth.make_st("tiny6", 0)
    m = runtime.Model(st, max_batch=4, token_chunk_size=128)
    try:
        m.infer_raw([0, 1], [2, 1], [5, 7, 9], [LAST, LAST])
        with pytest.raises(capi.B200Error) as e:
            m.debug_read("a_x2_lo", 3)
        assert e.value.code == capi.ERR_STATE
        assert m.debug_read("a_x2", 3).shape == (3, 256)
    finally:
        m.close()
    m = runtime.Model(st, max_batch=4, token_chunk_size=128, exact=True)
    try:
        m.infer_raw([0, 1], [2, 1], [5, 7, 9], [LAST, LAST])
        hi, lo = m.debug_read("a_x2", 3), m.debug_read("a_x2_lo", 3)
        assert np.array_equal(hi.astype(np.float16).astype(np.float32), hi)
        assert np.any(lo != 0) and np.all(np.abs(lo) <= np.abs(hi) * 2.0 ** -11 + 2.0 ** -24)
        with pytest.raises(capi.B200Error):
            m.debug_read("x_a_lo", 3)
    finally:
        m.close()
