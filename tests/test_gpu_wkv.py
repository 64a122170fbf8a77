"""The WKV kernel (csrc/wkv.cuh) driven alone through b200rwkv_op_wkv -- the step's own metadata (fill_meta), launch
(launch_wkv: kernel per version and output form, grid (H, min(S, rows)), th = 16 / 32 / 64 / 128) and decay fold operands --
against a float64 reference of the same operation, in the launch configurations the engine runs.

Reference (the model math of oracle/rwkv_numpy.py: _att_v56, _att_v7, wkv6_seq, wkv7_seq), in float64 from the exact f32 / f16
values the kernel receives:
  v5 / v6   o_t = sum_k r_k (u_k k_k v + M_{t-1}[., k]),  M_t = k v^T (as M[value][key]) + w M_{t-1};
            v6 fold: w = exp(-exp(bias + sum_k Wd2[c, k] d^_k)), d^ the f16-rounded d1 or hi + lo with precision 1;
  v7        kk = normalize_head(k k_k) with the 1e-12 clamp, k <- k (1 + (a - 1) k_a), v <- v + (v_first - v) nu after
            layer 0, sa = M_{t-1} (-kk), M_t = M_{t-1} w + sa (kk a)^T + v k^T, o_t = M_t r, bonus = sum_head(r k r_k);
  then GroupNorm over each head (eps 64e-5), * lnx_w + lnx_b, + bonus v (v7), * g.

Bound, per element, carried next to the reference rather than a flat tolerance (EPS = 2^-24, the f32 unit roundoff):
  * v5 / v6: magnitude recurrence  A_t = |k v^T| + w A_{t-1},  A_0 = |M_0|;  state error  E_t = (w + dw) E_{t-1} +
    C_STATE EPS A_t + dw A_{t-1}, dw the error of a folded decay (0 otherwise), so without the fold E_t <= C_STATE EPS t A_t;
    pre-norm output  |do| <= sum_k |r_k| (E_{t-1} + C_OUT EPS (A_{t-1} + |u k v|));
  * v7: the magnitude of one update  A_t = |M~_{t-1}| w + (|M~_{t-1}| |kk|) (x) |kk a| + |v| |k|^T  (|v|, |k| the magnitudes of
    the mixed operands, M~ the reference state widened by its error).  Carried elementwise from step to step this recurrence
    grows geometrically (its transition w + |kk| |kk a| has spectral radius up to 1.5) and says nothing after a few dozen
    tokens, so the error of each state row is carried as a 2-norm through the exact transition instead:
    e_t = e_{t-1} ||diag(w) - kk (kk a)^T||_2 + C_STATE EPS ||A_t row||_2, and |do| <= e_t ||r||_2 + C_OUT EPS sum |M~_t| |r|;
  * folded decay: the f32 dot product over Dd has error <= (Dd/2 + 2) EPS (sum |Wd2 d^| + |bias|), each expf 4 EPS relative,
    carried through exp(-exp(.));
  * GroupNorm: the mean, the variance (2 |d| dd + dd^2), rstd = 1/sqrt(var + eps) evaluated at the worst end of the interval,
    the normalised value, ln_x weight and bias; the v7 bonus (C_BONUS EPS sum |r| |k| |r_k|) times v; the gate;
  * precision 0 outputs add one f16 ulp of the reference (which saturates at +-65504); precision 1 outputs (hi + lo) add
    2^-22 |y| + 2^-25 (lo below the f16 normal range), and above 65504, where hi saturates and lo carries the rest,
    2^-11 (|y| - 65504); the pair saturates at +-131008.
Constants: C_STATE = 8 (v5 / v6) or 64 (v7, whose kk carries a normalisation), C_OUT = 16, C_BONUS = 16.  Every case prints
its worst error / bound for the outputs and the state; a ratio above 1 fails.

Beyond values: every pool slot not in the step keeps its NaN sentinel bit for bit, output rows the step does not own keep
theirs (rows T..rows-1, or T..15 and 16+T..31 with split output), layer 0 writes v_first = v bit for bit and later layers leave
it alone, and one sequence run as one launch or cut into launches of other shapes, slots and entry positions gives bit-identical
outputs and state (every path -- staged runs of <= 4 tokens, per-token runs, the per-token fold -- runs the same arithmetic).
"""
import dataclasses
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
GN_EPS = 64e-5
L2_EPS = 1e-12
C_STATE = {5: 8, 6: 8, 7: 64}
C_OUT = 16
C_BONUS = 16
V7_DECAY = 0.606531
F16_MAX = 65504.0
SENT32 = np.uint32(0x7FA5A5A5)      # NaN bit patterns no arithmetic produces
SENT16 = np.uint16(0x7E5A)
PER_TOKEN = ("r", "k", "v", "g", "w", "a", "nu", "v_first", "d1")


@dataclasses.dataclass(frozen=True)
class Case:
    version: int
    entries: tuple                  # ((pool slot, tokens), ...) in step order
    H: int = 4
    S: int = 0                      # 0: one more than the largest slot id
    Dd: int = 0                     # v6 decay fold rank (0: per-token decays)
    precision: int = 0
    layer: int = 0                  # v7: > 0 runs layer 0 first and feeds the v_first it wrote
    edge: str = ""

    @property
    def pool(self):
        return self.S or max(s for s, _ in self.entries) + 1


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def f32(x):
    return np.asarray(x, np.float32)


def sentinel32(shape):
    return np.full(shape, SENT32, np.uint32).view(np.float32)


def make_inputs(c: Case, rng, layer=0, v_first=None):
    """Per-channel parameters distinct per head and channel, per-token rows of the whole step."""
    H, C = c.H, c.H * 64
    T = sum(n for _, n in c.entries)
    head = lambda lo, hi: np.repeat(np.linspace(lo, hi, H), 64)
    ch = dict(lnx_w=f32(rng.uniform(-2, 2, C)), lnx_b=f32(rng.uniform(-1, 1, C)))
    tok = dict(r=f32(rng.standard_normal((T, C))), k=f32(rng.standard_normal((T, C)) * 0.5), v=f32(rng.standard_normal((T, C))),
               g=f32(rng.uniform(-1.5, 1.5, (T, C))))
    if c.version != 7:
        ch["u"] = f32(rng.standard_normal(C) * 0.5 + head(-0.5, 0.5))
    if c.version == 5:
        ch["w"] = f32(np.exp(-np.exp(head(-2.5, 0.5) + 0.5 * rng.standard_normal(C))))
    elif c.version == 6 and not c.Dd:
        tok["w"] = f32(np.exp(-np.exp(head(-2.5, 0.5) + 0.5 * rng.standard_normal((T, C)))))
    elif c.version == 6:
        tok["d1"] = f32(np.tanh(rng.standard_normal((T, c.Dd))))
        ch["time_decay_w2"] = (rng.standard_normal((C, c.Dd)) / np.sqrt(c.Dd)).astype(np.float16)
        ch["decay_bias"] = f32(head(-2.5, 0.5) + 0.3 * rng.standard_normal(C))
    else:
        tok["w"] = f32(np.exp(-V7_DECAY * sigmoid(rng.standard_normal((T, C)) + head(-2, 2))))
        tok["a"] = f32(sigmoid(rng.standard_normal((T, C))))
        ch.update(k_k=f32(rng.uniform(0.2, 1.5, C)), k_a=f32(rng.uniform(0, 1, C)), r_k=f32(rng.standard_normal(C) * 0.5 + head(-0.3, 0.3)))
        if layer:
            tok["nu"] = f32(sigmoid(rng.standard_normal((T, C))))
            tok["v_first"] = v_first.copy()
        else:
            tok["v_first"] = sentinel32((T, C))
    e = c.edge
    if e == "slow":                 # decay 1 - 2^-20: the state grows over the whole run
        if "w" in ch:
            ch["w"][:] = 1 - 2.0 ** -20
        else:
            tok["w"][:] = 1 - 2.0 ** -20
    if e == "zero_decay":           # head 0 forgets at once; the fold bias drives exp(-exp) to 0
        if "decay_bias" in ch:
            ch["decay_bias"][:64] = 10.0
        elif "w" in ch:
            ch["w"][:64] = 0
        else:
            tok["w"][:, :64] = 0
    if e == "r0":                   # head 1: output constant, variance 0, y = lnx_b g
        tok["r"][:, 64:128] = 0
    if e == "kk0":                  # head 1: k . k_k = 0, kk must be 0 (not NaN)
        ch["k_k"][64:128] = 0
    if e == "sat":                  # head 0 beyond 131008, head 1 between 65504 and 131008
        ch["lnx_b"][:64] = np.where(np.arange(64) % 2, 6e4, -6e4)
        ch["lnx_b"][64:128] = 4.4e4
        tok["g"][:, :128] = 2.5
    return ch, tok


def decay_of(c: Case, ch, tok, t, split):
    """Decay [H, 64] of token t (over the key index) and its error bound."""
    H = c.H
    if c.version == 5:
        return ch["w"].astype(np.float64).reshape(H, 64), np.zeros((H, 64))
    if c.version == 7 or not c.Dd:
        return tok["w"][t].astype(np.float64).reshape(H, 64), np.zeros((H, 64))
    d = tok["d1"][t]
    hi = d.astype(np.float16)
    dhat = hi.astype(np.float64)
    if split:
        dhat = dhat + (d - hi.astype(np.float32)).astype(np.float16).astype(np.float64)
    W = ch["time_decay_w2"].astype(np.float64)
    b = ch["decay_bias"].astype(np.float64)
    z = b + W @ dhat
    dz = (c.Dd / 2 + 2) * EPS * (np.abs(W) @ np.abs(dhat) + np.abs(b))
    e1 = np.exp(z)
    w = np.exp(-e1)
    de1 = e1 * (np.expm1(dz) + 4 * EPS * np.exp(dz))
    dw = w * (np.expm1(de1) + 4 * EPS)
    return w.reshape(H, 64), dw.reshape(H, 64)


def reference(c: Case, ch, tok, state0, layer):
    """float64 outputs y [T, C], their bound (before the f16 hand-off), and the final state with its bound per step slot."""
    H, C, ver = c.H, c.H * 64, c.version
    T = sum(n for _, n in c.entries)
    split = c.precision == 1
    g64 = lambda name: tok[name].astype(np.float64)
    y, dy = np.zeros((T, C)), np.zeros((T, C))
    states = {}
    chv = lambda name: ch[name].astype(np.float64).reshape(H, 64)
    lw, lb = chv("lnx_w"), chv("lnx_b")
    t0 = 0
    for slot, n in c.entries:
        M = state0[slot].astype(np.float64)
        A = np.abs(M)
        E = np.zeros_like(M)
        for t in range(t0, t0 + n):
            r, k, v = (g64(x)[t].reshape(H, 64) for x in ("r", "k", "v"))
            w, dw = decay_of(c, ch, tok, t, split)
            ar = np.abs(r)
            if ver != 7:
                u = chv("u")
                kv = v[:, :, None] * k[:, None, :]                              # [h, value, key]
                o = np.einsum("hk,hvk->hv", r, u[:, None, :] * kv + M)
                do = np.einsum("hk,hvk->hv", ar, E + C_OUT * EPS * (A + np.abs(u[:, None, :] * kv)))
                M = kv + w[:, None, :] * M
                An = np.abs(kv) + w[:, None, :] * A
                E = (w + dw)[:, None, :] * E + dw[:, None, :] * A + C_STATE[ver] * EPS * An
                A = An
            else:
                a = g64("a")[t].reshape(H, 64)
                kk = k * chv("k_k")
                kk = kk / np.maximum(np.sqrt((kk * kk).sum(-1, keepdims=True)), L2_EPS)
                ka = chv("k_a")
                kmag = np.abs(k) * (1 + np.abs(a - 1) * np.abs(ka))
                k = k * (1 + (a - 1) * ka)
                if layer == 0:
                    vmag, dv = np.abs(v), 0.0
                else:
                    vf, nu = g64("v_first")[t].reshape(H, 64), g64("nu")[t].reshape(H, 64)
                    vmag = np.abs(v) + np.abs(vf - v) * np.abs(nu)
                    v = v + (vf - v) * nu
                    dv = 3 * EPS * vmag
                b = kk * a
                # magnitude of this step's terms, taken at the kernel's state (reference + its error)
                Mag = np.abs(M) + E
                An = Mag * w[:, None, :] + np.einsum("hvk,hk->hv", Mag, np.abs(kk))[:, :, None] * np.abs(b)[:, None, :] \
                    + vmag[:, :, None] * kmag[:, None, :]
                Tn = np.linalg.norm(np.eye(64) * w[:, None, :] - kk[:, :, None] * b[:, None, :], 2, axis=(1, 2))
                e_row = E[:, :, 0] * Tn[:, None] + C_STATE[ver] * EPS * np.sqrt((An * An).sum(-1))
                sa = np.einsum("hvk,hk->hv", M, -kk)
                M = M * w[:, None, :] + sa[:, :, None] * b[:, None, :] + v[:, :, None] * k[:, None, :]
                E = np.repeat(e_row[:, :, None], 64, axis=2)
                o = np.einsum("hvk,hk->hv", M, r)
                do = e_row * np.sqrt((r * r).sum(-1, keepdims=True)) + C_OUT * EPS * np.einsum("hvk,hk->hv", np.abs(M) + E, ar)
            # GroupNorm over each head, ln_x, bonus, gate
            mu = o.mean(-1, keepdims=True)
            d = o - mu
            var = (d * d).mean(-1, keepdims=True)
            s = var + GN_EPS
            rstd = 1 / np.sqrt(s)
            dmu = do.mean(-1, keepdims=True) + 8 * EPS * np.abs(o).mean(-1, keepdims=True)
            dd = do + dmu + EPS * np.abs(d)
            ds = (2 * np.abs(d) * dd + dd * dd).mean(-1, keepdims=True) + 8 * EPS * var + EPS * s
            assert np.all(s - ds > 0), "the variance bound swallows eps"
            drstd = 1 / np.sqrt(s - ds) - rstd + 3 * EPS * rstd
            nrm = d * rstd
            dn = dd * rstd + np.abs(d) * drstd + dd * drstd + EPS * np.abs(nrm)
            yy = nrm * lw + lb
            dyy = dn * np.abs(lw) + 2 * EPS * (np.abs(nrm * lw) + np.abs(yy))
            if ver == 7:
                rk = chv("r_k")
                bonus = (r * k * rk).sum(-1, keepdims=True)
                dbonus = C_BONUS * EPS * (ar * kmag * np.abs(rk)).sum(-1, keepdims=True)
                yy = yy + bonus * v
                dyy = dyy + dbonus * np.abs(v) + (np.abs(bonus) + dbonus) * dv + EPS * (np.abs(bonus * v) + np.abs(yy))
            gg = g64("g")[t].reshape(H, 64)
            y[t] = (yy * gg).reshape(C)
            dy[t] = (dyy * np.abs(gg) + EPS * np.abs(yy * gg)).reshape(C)
        states[slot] = (M, E)
        t0 += n
    return y, dy, states


def f16_ulp(x):
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14)))
    return 2.0 ** (e - 10)


def launch(c: Case, ch, tok, state, layer=0, **snap):
    """One b200rwkv_op_wkv call with sentinel-filled outputs; state [S, H, 64, 64] and tok["v_first"] are updated in place.
    `snap`: op_wkv_step's snapshot arguments."""
    T = sum(n for _, n in c.entries)
    out = np.full((capi.gemm_rows(T, c.precision), c.H * 64), SENT16, np.uint16)
    kw = {n: x for n, x in tok.items() if n != "v_first"}
    kw.update(ch)
    if c.version == 7:
        kw["v_first"] = tok["v_first"]
        kw["layer0"] = layer == 0
    capi.op_wkv_step(c.version, [s for s, _ in c.entries], [n for _, n in c.entries], state, out, precision=c.precision, **kw,
                     **snap)
    return out


def check(name, c: Case, rng, layer=0, v_first=None):
    """Run one launch of case c and hold it to the reference; returns the v_first it leaves (v7)."""
    H, C, S = c.H, c.H * 64, c.pool
    T = sum(n for _, n in c.entries)
    ch, tok = make_inputs(c, rng, layer, v_first)
    state = sentinel32((S, H, 64, 64))
    for s, _ in c.entries:
        state[s] = f32(rng.standard_normal((H, 64, 64)) * 0.3)
    state0 = state.copy()
    vf_in = tok["v_first"].copy() if c.version == 7 else None
    out = launch(c, ch, tok, state, layer)

    y, dy, states = reference(c, ch, tok, state0, layer)
    # outputs
    if c.precision == 0:
        got = out[:T].view(np.float16).astype(np.float64)
        want = np.clip(y, -F16_MAX, F16_MAX)
        bound = dy + f16_ulp(want)
        own = np.arange(T)
    else:
        hi, lo = out[:T].view(np.float16), out[16:16 + T].view(np.float16)
        assert np.all(np.isfinite(hi)) and np.all(np.isfinite(lo)), f"{name}: an infinite split half"
        got = hi.astype(np.float64) + lo.astype(np.float64)
        want = np.clip(y, -2 * F16_MAX, 2 * F16_MAX)
        bound = dy + 2.0 ** -22 * np.abs(want) + 2.0 ** -11 * np.maximum(np.abs(want) - F16_MAX, 0) + 2.0 ** -25
        own = np.concatenate([np.arange(T), 16 + np.arange(T)])
    err = np.abs(got - want)
    ratio_out = float(np.max(np.where(np.isnan(err), np.inf, err / bound)))
    # state of every slot of the step
    ratio_state = 0.0
    for s, (M, E) in states.items():
        e = np.abs(state[s].astype(np.float64) - M)
        ratio_state = max(ratio_state, float(np.max(np.where(np.isnan(e), np.inf, e / (E + EPS * np.abs(M) + 1e-30)))))
    print(f"\n[wkv] {name} layer {layer}: worst |err|/bound out {ratio_out:.4f} state {ratio_state:.4f}")
    assert ratio_out <= 1.0, f"{name}: output error / bound {ratio_out}"
    assert ratio_state <= 1.0, f"{name}: state error / bound {ratio_state}"
    # what the step must leave alone
    rest = [s for s in range(S) if s not in states]
    assert np.array_equal(state[rest].view(np.uint32), state0[rest].view(np.uint32)), f"{name}: a slot outside the step changed"
    mask = np.ones(out.shape[0], bool)
    mask[own] = False
    assert np.all(out[mask] == SENT16), f"{name}: an output row the step does not own was written"
    if c.version == 7:
        if layer == 0:
            assert np.array_equal(tok["v_first"].view(np.uint32), tok["v"].view(np.uint32)), f"{name}: v_first != v"
        else:
            assert np.array_equal(tok["v_first"].view(np.uint32), vf_in.view(np.uint32)), f"{name}: a later layer wrote v_first"
        return tok["v_first"]
    return None


def run(name, c: Case):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    vf = check(name, c, rng)
    if c.version == 7 and c.layer:
        check(name, c, rng, layer=c.layer, v_first=vf)


# ---- cases -------------------------------------------------------------------------------------------------------------
VERSIONS = {"v5": dict(version=5), "v6": dict(version=6), "v6fold64": dict(version=6, Dd=64), "v6fold128": dict(version=6, Dd=128),
            "v7": dict(version=7), "v7L1": dict(version=7, layer=1)}
# tokens in one slot: staged runs (<= 4), the first per-token run (5), and every th bucket (16 / 32 / 64 / 128) at both ends
COUNTS = (1, 2, 4, 5, 16, 17, 64, 65, 128)
BATCHES = {
    "ragged": dict(entries=((0, 5), (1, 1), (2, 4), (3, 7), (4, 3))),
    "sparse_permuted": dict(entries=((7, 2), (0, 5), (12, 1), (3, 3)), S=16),
    "dead_ctas": dict(entries=((30, 1), (2, 3)), S=32),
    "tp_local_heads": dict(entries=((1, 1), (0, 1), (3, 1), (2, 1)), H=32),
}
CASES = {}
for vn, vk in VERSIONS.items():
    for n in COUNTS:
        CASES[f"{vn}-one_slot_{n}"] = Case(entries=((0, n),), H=2, **vk)
    for bn, bk in BATCHES.items():
        CASES[f"{vn}-{bn}"] = Case(**bk, **vk)
    # split output: decode-shaped steps of <= 16 tokens, staged and per-token runs
    CASES[f"{vn}-split_decode"] = Case(entries=((2, 1), (0, 1), (5, 1)), precision=1, **vk)
    CASES[f"{vn}-split_ragged16"] = Case(entries=((1, 5), (3, 4), (0, 7)), precision=1, **vk)
    CASES[f"{vn}-r0_head"] = Case(entries=((0, 3), (1, 6)), edge="r0", **vk)
    CASES[f"{vn}-saturate"] = Case(entries=((0, 2), (1, 5)), edge="sat", **vk)
    CASES[f"{vn}-split_overflow"] = Case(entries=((0, 2), (1, 5)), edge="sat", precision=1, **vk)
# the model launch shapes: 7B decode headline (16 slots of 1 token, 64 heads, Dd 128), RWKV-7 2.9B (40 heads, 8 slots),
# one 3B slot (40 heads, Dd 64)
CASES["v6fold128-7b_decode16"] = Case(version=6, Dd=128, H=64, entries=tuple((s, 1) for s in range(16)))
CASES["v6fold128-7b_decode16_split"] = Case(version=6, Dd=128, H=64, entries=tuple((s, 1) for s in range(16)), precision=1)
CASES["v7L1-2.9b_decode8"] = Case(version=7, layer=1, H=40, entries=tuple((s, 1) for s in (3, 0, 7, 1, 6, 2, 5, 4)))
CASES["v6fold64-3b_one_slot"] = Case(version=6, Dd=64, H=40, entries=((0, 1),))
CASES["v6fold64-3b_prefill"] = Case(version=6, Dd=64, H=40, entries=((0, 33),))
CASES["v5-slow_decay_128"] = Case(version=5, H=2, entries=((0, 128),), edge="slow")
CASES["v6-slow_decay_128"] = Case(version=6, H=2, entries=((0, 128),), edge="slow")
for vn in ("v5", "v6", "v6fold64"):
    CASES[f"{vn}-zero_decay"] = Case(entries=((0, 3), (1, 6)), edge="zero_decay", **VERSIONS[vn])
CASES["v7-kk0_head"] = Case(version=7, entries=((0, 3), (1, 6)), edge="kk0")
CASES["v7L1-kk0_head_split"] = Case(version=7, layer=1, entries=((0, 3), (1, 6)), edge="kk0", precision=1)


@pytest.mark.parametrize("name", list(CASES))
def test_wkv_matches_float64_reference(name):
    run(name, CASES[name])


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("vn", ["v5", "v6", "v6fold64", "v7L1"])
def test_wkv_cut_into_other_launches_is_bit_identical(vn, precision):
    """One sequence of 13 tokens as one launch (a per-token run), and as launches of 1 + 4 + 5 + 3 tokens in other slots and
    entry positions, next to other sequences (staged and per-token runs, th 16 / 32 / 64), the state carried between
    launches: outputs and the final state are identical bit for bit."""
    vk = VERSIONS[vn]
    H, N = 2, 13
    rng = np.random.default_rng(zlib.crc32(f"chain {vn} {precision}".encode()))
    layer = vk.get("layer", 0)
    whole = Case(entries=((3, N),), H=H, S=8, precision=precision, **vk)
    ch, tok = make_inputs(whole, rng, layer, f32(rng.standard_normal((N, H * 64))))
    M0 = f32(rng.standard_normal((H, 64, 64)) * 0.3)
    state = np.zeros((8, H, 64, 64), np.float32)
    state[3] = M0
    t = {n: x.copy() for n, x in tok.items()}
    out = launch(whole, ch, t, state, layer)
    want_out = out[:N] if precision == 0 else np.concatenate([out[:N], out[16:16 + N]])
    want_state = state[3].copy()

    # (sequence slot, sequence tokens, fillers before it [(slot, n)], fillers after it)
    if precision == 0:
        plan = [(0, 1, [(5, 2)], []), (6, 4, [], []), (7, 5, [(1, 3), (2, 20)], []), (4, 3, [], [(5, 30)])]
    else:
        plan = [(0, 1, [(5, 2)], [(1, 4)]), (6, 4, [], []), (7, 5, [(1, 3), (2, 5)], []), (4, 3, [], [(5, 1)])]
    state = np.zeros((8, H, 64, 64), np.float32)
    cur, at, outs = None, 0, []
    for slot, n, before, after in plan:
        state[slot] = M0 if cur is None else state[cur]
        entries = tuple(before) + ((slot, n),) + tuple(after)
        c = Case(entries=entries, H=H, S=8, precision=precision, **vk)
        _, filler = make_inputs(c, rng, layer, f32(rng.standard_normal((sum(m for _, m in entries), H * 64))))
        # the sequence's rows go where its entry sits in this step
        r0 = sum(m for _, m in before)
        for key in filler:
            filler[key][r0:r0 + n] = tok[key][at:at + n]
        o = launch(c, ch, filler, state, layer)
        outs.append(o[r0:r0 + n] if precision == 0 else np.concatenate([o[r0:r0 + n], o[16 + r0:16 + r0 + n]]))
        cur, at = slot, at + n
    if precision == 0:
        got_out = np.concatenate(outs)
    else:
        got_out = np.concatenate([np.concatenate([o[:len(o) // 2] for o in outs]), np.concatenate([o[len(o) // 2:] for o in outs])])
    assert np.array_equal(got_out, want_out)
    assert np.array_equal(state[cur].view(np.uint32), want_state.view(np.uint32))
