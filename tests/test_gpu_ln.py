"""The LN stages (csrc/mix.cuh: embed_ln0_kernel, ln_mix_kernel, ln_out_kernel; csrc/pre6.cuh: ln_mix_cluster_kernel and the
RWKV-6 front half pre6_kernel) driven alone through b200rwkv_op_ln -- the step's own metadata (fill_meta), parameter blocks
and launch (launch_embed / launch_ln / launch_pre6 / launch_ln_out: kernel choice, cluster and PDL attributes, token rows of
the operands) -- against a float64 reference of the same operation, in the launch configurations the engine runs.

Reference, in float64 from the exact f32 / f16 values the kernel receives:
  residual  a = x + g (.) sum_p part_p, g the gate block of column c (1 without gates);
  LN        mu = mean(a), var = mean((a - mu)^2), xx = (a - mu) / sqrt(var + 1e-5) w + b;
  shift     prev = shift_state[slot] for an entry's first token, else the LN of the previous token's residual;
            sx = prev - xx, mix_j = xx + sx mu_j;
  embed     LN0 of f32(emb[token]);  ln_out: head row r(t) = LN(a), hidden row = a;
  front half, checked in stages from the kernel's own intermediates so that a failure names its phase:
            phase 1 as above; phase 2  lora = tanh(W1 x^), x^ the kernel's own f16 (or hi + lo) mix-0 output;
            phase 3  out_j = xx + sx (mu5_j + W2_j lora^_j) from the kernel's own xx, sx and LoRA rows.

Bound, per element, carried next to the reference (EPS = 2^-24, the f32 unit roundoff):
  * residual: the f32 sum of the parts ((n_parts + 1) EPS sum |part| |g|), the gate multiply and the add;
  * the LN statistics of the kernel's own f32 residual row: the mean with D_MEAN = 24 + NV roundings (per-thread float4
    sums, NV vectors per thread, the 5-level warp tree twice over 8 warps, the 8-way slice combine of the cluster kernels,
    the division), the two-pass variance with D_MEAN + 4 plus the square of the mean's error and, for the cluster kernels'
    Chan combine, 2 max_i |mu_i - mu| (the slice means' error + the mean's error); rstd at the worst end of its interval
    plus 4 EPS; then the normalised value, w and b (3 EPS each);
  * f16 outputs add one f16 ulp of the reference (which saturates at +-65504); split outputs (hi + lo) add
    2^-22 |y| + 2^-25, and 2^-11 (|y| - 65504) above 65504 where lo carries the rest; the pair saturates at +-131008;
  * front half phase 2: tests/test_gpu_gemm.py's 2^-14 sum |x^ W1| carried through tanh (Lipschitz 1) plus 4 EPS; phase 3: the same
    2^-14 sum |W2 lora^| times |sx|, plus the f32 lerp.
Every case prints its worst error / bound per output; a ratio above 1 fails.

Beyond values, bit for bit: sentinels in every cell a stage must not write (mix, LoRA, front-half and head rows past the
step, split rows 16 + T .. 31, pool rows of slots outside the step, x_in of the in-place stage); committed rows equal to
commit_src of the entry's last token; hidden rows equal to x_out; three launches on inputs A, B, A with slices 0 and 2
identical (for pre6_kernel this re-arms its grid-barrier counters); an entry gives the same rows wherever it sits in the step;
pre6_kernel's phase 1 equal to ln_mix_cluster_kernel's; and the residual row of ln_mix_kernel (residual_row) equal to the
cluster kernels' (residual_vec).
"""
import dataclasses
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
LN_EPS = 1e-5
F16_MAX = 65504.0
SENT32 = np.uint32(0x7FA5A5A5)      # NaN bit patterns no arithmetic produces
SENT16 = np.uint16(0x7E5A)
STAGE = {"embed": capi.LN_EMBED, "ln": capi.LN_MIX, "pre6": capi.LN_FRONT6, "out": capi.LN_OUT}


@dataclasses.dataclass(frozen=True)
class Case:
    stage: str
    C: int
    entries: tuple                  # ((pool slot, tokens), ...) in step order
    S: int = 0                      # 0: one more than the largest slot id
    n_parts: int = 1
    n_gate: int = 1
    n_mix: int = 2
    precision: int = 0
    Dm: int = 32
    options: tuple = ()             # ln_out: capi.OPTION_* per entry (default LAST)
    commit: bool = True
    hidden: bool = True
    in_place: bool = False          # LN1 of layer 0: x_out is x_in
    edge: str = ""
    kernel: int = -1                # kernel the case must run (capi.K_*)

    @property
    def pool(self):
        return self.S or max(s for s, _ in self.entries) + 1

    @property
    def T(self):
        return sum(n for _, n in self.entries)

    @property
    def rows(self):                 # token rows of the A16 operands
        return capi.gemm_rows(self.T, self.precision)


def f32(x):
    return np.asarray(x, np.float32)


def sentinel32(shape):
    return np.full(shape, SENT32, np.uint32).view(np.float32)


def f16_ulp(x):
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -14)))
    return 2.0 ** (e - 10)


def ratio(got, want, bound):
    err = np.abs(np.asarray(got, np.float64) - want)
    return float(np.max(np.where(np.isnan(err), np.inf, err / bound), initial=0.0))


def f16_got(bits, want, dy, split, T):
    """Value of an f16 (or hi + lo) operand [..., rows, K] for T tokens, with the clipped reference and the bound."""
    if not split:
        got = bits[..., :T, :].view(np.float16).astype(np.float64)
        w = np.clip(want, -F16_MAX, F16_MAX)
        return got, w, dy + f16_ulp(w)
    hi, lo = bits[..., :T, :].view(np.float16), bits[..., 16:16 + T, :].view(np.float16)
    assert np.all(np.isfinite(hi)) and np.all(np.isfinite(lo)), "an infinite split half"
    got = hi.astype(np.float64) + lo.astype(np.float64)
    w = np.clip(want, -2 * F16_MAX, 2 * F16_MAX)
    return got, w, dy + 2.0 ** -22 * np.abs(w) + 2.0 ** -11 * np.maximum(np.abs(w) - F16_MAX, 0) + 2.0 ** -25


def own_rows(T, split):
    return list(range(T)) + (list(range(16, 16 + T)) if split else [])


# ---- inputs ----------------------------------------------------------------------------------------------------------
def entry_rows(c: Case, slot, n, variant):
    """Per-token inputs of one entry, from a generator seeded by (case shape, slot, variant): the same entry gets the same
    rows wherever it sits in a step."""
    rng = np.random.default_rng([c.C, c.n_parts, c.n_gate, slot, variant, zlib.crc32(c.edge.encode())])
    C, gcl = c.C, (c.C // c.n_gate if c.n_gate else 0)
    d = dict(x_in=rng.standard_normal((n, C)) * 2 + rng.standard_normal(C),
             parts=rng.standard_normal((c.n_parts, n, C)) * 0.5,
             gates=rng.uniform(-1.5, 1.5, (c.n_gate, n, gcl)),
             commit_src=rng.standard_normal((n, C)),
             tokens=rng.integers(0, 1000, n),
             shift=rng.standard_normal(C))
    if c.edge == "const":           # sigma^2 = 0 in every row
        d["x_in"][:] = 0.75
        d["parts"][:] = 0
    if c.edge == "big":             # 1e4 + N(0, 1): a one-pass E[x^2] - mu^2 variance loses every digit
        d["x_in"] = 1e4 + rng.standard_normal((n, C))
        d["parts"] *= 0.01
    if c.edge == "slices":          # the eight channel slices of the cluster kernels sit far apart
        d["x_in"] += np.repeat(np.array([300.0, -250, 40, -1000, 600, 5, -75, 900]), C // 8)
    if c.edge == "embed_ends":
        d["tokens"][:] = np.where(np.arange(n) % 2, 999, 0)
    return {k: (v if k == "tokens" else f32(v)) for k, v in d.items()}


def make_inputs(c: Case, variants):
    """Inputs of len(variants) launches: per-token arrays [launches, ...], parameters shared by every launch."""
    C, S, T = c.C, c.pool, c.T
    rng = np.random.default_rng([c.C, c.n_mix, c.Dm, zlib.crc32(c.edge.encode())])
    per = [[entry_rows(c, s, n, v) for s, n in c.entries] for v in variants]
    cat = lambda k, ax: np.stack([np.concatenate([e[k] for e in launch], axis=ax) for launch in per])
    x = dict(x_in=cat("x_in", 0), parts=cat("parts", 1), gates=cat("gates", 1), commit_src=cat("commit_src", 0),
             tokens=cat("tokens", 0).astype(np.uint32))
    x["ln_w"] = f32(rng.uniform(-2, 2, C))
    x["ln_b"] = f32(rng.uniform(-1, 1, C))
    x["shift_state"] = sentinel32((S, C))           # shared by the launches: the first launch's rows
    for (s, _), e in zip(c.entries, per[0]):
        x["shift_state"][s] = e["shift"]
    x["mu"] = f32(rng.uniform(-0.5, 1.5, (c.n_mix, C)))          # inside and outside [0, 1]
    if c.edge == "w0":
        x["ln_w"][:] = 0
    if c.edge == "sat":             # mixes past 65504 and past 131008, sx up to ~1e5
        x["ln_b"][: C // 2] = np.where(np.arange(C // 2) % 2, 6e4, -6e4)
        for s, _ in c.entries:
            x["shift_state"][s, : C // 4] = 1e5
        x["mu"][:, : C // 4] = np.linspace(-1.5, 2.5, C // 4)
    if c.stage == "pre6":
        Dm = c.Dm
        x["W1"] = (rng.standard_normal((5 * Dm, C)) / np.sqrt(C) * 3).astype(np.float16)
        x["W2"] = (rng.standard_normal((5, C, Dm)) / np.sqrt(Dm)).astype(np.float16)
        x["mu5"] = f32(rng.uniform(-0.5, 1.5, (5, C)))
        if c.edge == "sat":
            x["mu5"][:, : C // 4] = 2.5
    if c.stage == "embed":
        x["emb"] = (rng.standard_normal((1000, C)) * 0.3 + rng.standard_normal((1000, 1))).astype(np.float16)
    return x


def run_op(c: Case, x, launches, **snap):
    """One b200rwkv_op_ln call with sentinel-filled outputs; returns the outputs and the kernel report.  `snap`: op_ln's
    snapshot arguments."""
    C, S, T, R = c.C, c.pool, c.T, c.rows
    L = launches
    o = dict(commit_dst=sentinel32((S, C)) if c.commit else None)
    kw = dict(S=S, ln_w=x["ln_w"], ln_b=x["ln_b"])
    if c.stage == "embed":
        o["x_out"] = sentinel32((L, T, C))
        kw.update(emb=x["emb"].view(np.uint16), V=x["emb"].shape[0], tokens=np.ascontiguousarray(x["tokens"]))
        o.pop("commit_dst")
    else:
        kw.update(x_in=x["x_in"].copy(), n_parts=c.n_parts, n_gate=c.n_gate,
                  parts=x["parts"] if c.n_parts else None, gates=x["gates"] if c.n_gate else None,
                  commit_src=x["commit_src"] if c.commit else None)
        o["hidden"] = sentinel32((L, T, C)) if c.hidden else None
    option = None
    if c.stage in ("ln", "pre6"):
        kw.update(shift_state=x["shift_state"], n_mix=c.n_mix, mu=x["mu"])
        o.update(x_out=None if c.in_place else sentinel32((L, T, C)), xx_out=sentinel32((L, T, C)), sx_out=sentinel32((L, T, C)),
                 mix_out=np.full((L, c.n_mix, R, C), SENT16, np.uint16))
    if c.stage == "pre6":
        kw.update(Dm=c.Dm, W1=x["W1"].view(np.uint16), W2=x["W2"].view(np.uint16), mu5=x["mu5"])
        o.update(lora_out=np.full((L, 5, R, c.Dm), SENT16, np.uint16), out5=np.full((L, 5, R, C), SENT16, np.uint16))
    if c.stage == "out":
        option = list(c.options) or [capi.OPTION_LAST] * len(c.entries)
        nr = sum(n if op == capi.OPTION_FULL else (1 if op == capi.OPTION_LAST else 0) for (_, n), op in zip(c.entries, option))
        hr = 32 if c.precision else capi.gemm_rows(max(nr, 1))
        o["head_out"] = np.full((L, hr, C), SENT16, np.uint16)
    kern = capi.op_ln(STAGE[c.stage], C, [s for s, _ in c.entries], [n for _, n in c.entries], launches=L,
                      precision=c.precision, option=option, **kw, **o, **snap)
    o["x_in_after"] = kw.get("x_in")
    return o, kern, option


# ---- reference -------------------------------------------------------------------------------------------------------
def nv_of(C):
    nv = -(-C // 1024)
    return 1 if nv <= 1 else 2 if nv == 2 else 4 if nv <= 4 else 8


def residual_ref(c: Case, x, l):
    """float64 a = x + g (.) sum parts of launch l, and its bound [T, C]."""
    a = x["x_in"][l].astype(np.float64)
    if not c.n_parts:
        return a, np.zeros_like(a)
    p = x["parts"][l].astype(np.float64)
    s, sa = p.sum(0), np.abs(p).sum(0)
    if c.n_gate:
        g = np.concatenate(list(x["gates"][l].astype(np.float64)), axis=1)      # [T, C]: block q holds columns q * C / n_gate ..
    else:
        g = np.ones_like(s)
    y = a + g * s
    return y, 2 * EPS * ((c.n_parts + 1) * np.abs(g) * sa + np.abs(a) + np.abs(g * s) + np.abs(y))


def ln_ref(a, w, b, C, cluster):
    """LN of rows a [n, C] (the kernel's own f32 values) and its bound."""
    a = a.astype(np.float64)
    w, b = w.astype(np.float64), b.astype(np.float64)
    dm = 24 + nv_of(C)
    mu = a.mean(-1, keepdims=True)
    d = a - mu
    var = (d * d).mean(-1, keepdims=True)
    dmu = dm * EPS * np.abs(a).mean(-1, keepdims=True)
    sl = a.reshape(a.shape[0], 8, C // 8)
    dmu_s = dm * EPS * np.abs(sl).mean(-1).max(-1, keepdims=True)
    off = np.abs(sl.mean(-1) - mu).max(-1, keepdims=True)
    dvar = (dm + 4) * EPS * var + dmu * dmu + (2 * off * (dmu_s + dmu) + 2 * dmu_s * dmu_s if cluster else 0)
    r = 1 / np.sqrt(var + LN_EPS)
    r_hi = 1 / np.sqrt(np.maximum(var - dvar, 0) + LN_EPS)
    dr = np.maximum(r_hi - r, r - 1 / np.sqrt(var + dvar + LN_EPS)) + 4 * EPS * r_hi
    n = d * r
    dn = (np.abs(d) + dmu) * dr + r * dmu + 3 * EPS * (np.abs(d) + dmu) * (r + dr)
    y = n * w + b
    return y, np.abs(w) * dn + 3 * EPS * (np.abs(n * w) + np.abs(b) + np.abs(y))


def first_of_entry(c: Case):
    first, slot_of, last = [], [], []
    for s, n in c.entries:
        first += [True] + [False] * (n - 1)
        slot_of += [s] * n
        last += [False] * (n - 1) + [True]
    return np.array(first), np.array(slot_of), np.array(last)


def check_ln_launch(name, c: Case, x, o, l, worst):
    """Residual, LN, shift and mixes of launch l of an LN / front-half stage; returns (xx, sx) the kernel wrote."""
    T, C = c.T, c.C
    cluster = c.T <= 16
    split = c.precision == 1
    a_ref, da = residual_ref(c, x, l)
    a_k = x["x_in"][l] if c.in_place else o["x_out"][l]
    worst["x_out"] = max(worst.get("x_out", 0), ratio(a_k, a_ref, da + 1e-300))
    xx, dxx = ln_ref(a_k, x["ln_w"], x["ln_b"], C, cluster)
    first, slot_of, _ = first_of_entry(c)
    prev = np.where(first[:, None], x["shift_state"][slot_of].astype(np.float64), np.roll(xx, 1, 0))
    dprev = np.where(first[:, None], 0.0, np.roll(dxx, 1, 0))
    sx = prev - xx
    dsx = dprev + dxx + EPS * np.abs(sx)
    worst["xx"] = max(worst.get("xx", 0), ratio(o["xx_out"][l], xx, dxx))
    worst["sx"] = max(worst.get("sx", 0), ratio(o["sx_out"][l], sx, dsx))
    for j in range(c.n_mix):
        m = x["mu"][j].astype(np.float64)
        y = xx + sx * m
        dy = dxx + np.abs(m) * dsx + 2 * EPS * (np.abs(sx * m) + np.abs(y))
        got, want, bound = f16_got(o["mix_out"][l, j], y, dy, split, T)
        worst[f"mix{j}"] = max(worst.get(f"mix{j}", 0), ratio(got, want, bound))
    if c.stage == "pre6":
        check_pre6_launch(c, x, o, l, worst)


def check_pre6_launch(c: Case, x, o, l, worst):
    """Phases 2 and 3 of the front half from the kernel's own mix-0, xx, sx and LoRA rows."""
    T, Dm, split = c.T, c.Dm, c.precision == 1
    val = lambda bits: bits[..., :T, :].view(np.float16).astype(np.float64) + (
        bits[..., 16:16 + T, :].view(np.float16).astype(np.float64) if split else 0)
    xh = val(o["mix_out"][l, 0])                                  # [T, C]
    W1 = x["W1"].astype(np.float64)                               # [5 Dm, C]
    z = xh @ W1.T
    dz = 2.0 ** -14 * (np.abs(xh) @ np.abs(W1).T)
    lora = np.tanh(z)
    dl = dz + 4 * EPS * np.abs(lora)
    lora5 = lora.reshape(T, 5, Dm).transpose(1, 0, 2)
    dl5 = dl.reshape(T, 5, Dm).transpose(1, 0, 2)
    got, want, bound = f16_got(o["lora_out"][l], lora5, dl5, split, T)
    worst["lora"] = max(worst.get("lora", 0), ratio(got, want, bound))
    lh = val(o["lora_out"][l])                                    # [5, T, Dm]
    xx, sx = o["xx_out"][l].astype(np.float64), o["sx_out"][l].astype(np.float64)
    for j in range(5):
        W2 = x["W2"][j].astype(np.float64)                        # [C, Dm]
        yl = lh[j] @ W2.T
        dyl = 2.0 ** -14 * (np.abs(lh[j]) @ np.abs(W2).T)
        m = x["mu5"][j].astype(np.float64) + yl
        y = xx + sx * m
        dy = np.abs(sx) * (dyl + EPS * np.abs(m)) + 2 * EPS * (np.abs(sx * m) + np.abs(y))
        got, want, bound = f16_got(o["out5"][l, j], y, dy, split, T)
        worst["out5"] = max(worst.get("out5", 0), ratio(got, want, bound))


def check_bits(name, c: Case, x, o, L):
    """Cells the stage must not write keep their sentinels; commits and hidden rows are exact copies."""
    T, split = c.T, c.precision == 1
    if c.stage in ("ln", "pre6"):
        keep = np.ones(c.rows, bool)
        keep[own_rows(T, split)] = False
        assert np.all(o["mix_out"][:, :, keep] == SENT16), f"{name}: a mix row past the step was written"
        if c.stage == "pre6":
            assert np.all(o["lora_out"][:, :, keep] == SENT16), f"{name}: a LoRA row past the step was written"
            assert np.all(o["out5"][:, :, keep] == SENT16), f"{name}: a front-half row past the step was written"
        if c.in_place:
            assert np.array_equal(o["x_in_after"].view(np.uint32), x["x_in"].view(np.uint32)), f"{name}: x_in changed in place"
    if c.stage != "embed" and c.hidden:
        src = x["x_in"] if c.in_place else (o["x_out"] if "x_out" in o and o["x_out"] is not None else None)
        if src is not None:
            assert np.array_equal(o["hidden"].view(np.uint32), src.view(np.uint32)), f"{name}: hidden rows != x_out"
    if c.commit and c.stage != "embed":
        _, slot_of, last = first_of_entry(c)
        want = sentinel32((c.pool, c.C))
        want[slot_of[last]] = x["commit_src"][L - 1][last]
        assert np.array_equal(o["commit_dst"].view(np.uint32), want.view(np.uint32)), f"{name}: commit_dst"


def check_out_launch(name, c: Case, x, o, l, option, worst):
    T, C, split = c.T, c.C, c.precision == 1
    a_ref, da = residual_ref(c, x, l)
    a_k = o["hidden"][l] if c.hidden else a_ref
    if c.hidden:
        worst["hidden"] = max(worst.get("hidden", 0), ratio(a_k, a_ref, da + 1e-300))
    y, dy = ln_ref(a_k, x["ln_w"], x["ln_b"], C, False)
    if not c.hidden:                # the kernel's residual is not visible: carry its bound through the LN (|dLN/da| <= 2 r |w|)
        r = 1 / np.sqrt(((a_ref - a_ref.mean(-1, keepdims=True)) ** 2).mean(-1, keepdims=True) + LN_EPS)
        dy = dy + 2 * r * np.abs(x["ln_w"]) * (da + da.mean(-1, keepdims=True))
    outrow = []
    for (s, n), op in zip(c.entries, option):
        outrow += [op == capi.OPTION_FULL or (op == capi.OPTION_LAST and j == n - 1) for j in range(n)]
    toks = np.nonzero(outrow)[0]
    Rn = len(toks)
    head = o["head_out"][l]
    got, want, bound = f16_got(head, y[toks], dy[toks], split, Rn)
    worst["head"] = max(worst.get("head", 0), ratio(got, want, bound))
    keep = np.ones(head.shape[0], bool)
    keep[own_rows(Rn, split)] = False
    assert np.all(head[keep] == SENT16), f"{name}: a head row past the logits rows was written"


def run_case(name, c: Case, variants=(0,)):
    """Run the stage over len(variants) launches, hold every launch to the reference, return the outputs."""
    L = len(variants)
    x = make_inputs(c, variants)
    o, kern, option = run_op(c, x, L)
    if c.kernel >= 0:
        assert kern[0] == c.kernel, f"{name}: ran kernel {kern}, expected {c.kernel}"
    assert kern[2] == c.precision or c.stage == "embed", f"{name}: split {kern[2]}"
    worst = {}
    for l in range(L):
        if c.stage == "embed":
            e = x["emb"][x["tokens"][l]].astype(np.float32)
            y, dy = ln_ref(e, x["ln_w"], x["ln_b"], c.C, False)
            worst["x_out"] = max(worst.get("x_out", 0), ratio(o["x_out"][l], y, dy))
        elif c.stage == "out":
            check_out_launch(name, c, x, o, l, option, worst)
        else:
            check_ln_launch(name, c, x, o, l, worst)
    check_bits(name, c, x, o, L)
    print(f"\n[ln] {name} kernel {kern}: " + " ".join(f"{k} {v:.4f}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, f"{name}: {k} error / bound {v}"
    return x, o, kern


# ---- cases -------------------------------------------------------------------------------------------------------------
K = dict(ln=capi.K_LN_MIX, cl=capi.K_LN_MIX_CLUSTER, pre6=capi.K_PRE6, out=capi.K_LN_OUT, embed=capi.K_EMBED)
CASES = {}
# every NV of the per-token kernels and the partial CTA slices of the cluster kernel (C / 8 not a multiple of 128)
for C in (64, 256, 1024, 1088, 2048, 2560, 4096, 4160, 8192):
    CASES[f"cluster-C{C}-T15"] = Case("ln", C, ((3, 5), (0, 1), (9, 9)), kernel=K["cl"])
    CASES[f"cluster-C{C}-split"] = Case("ln", C, ((3, 1), (1, 1), (6, 1)), precision=1, kernel=K["cl"])
    CASES[f"mix-C{C}-T33"] = Case("ln", C, ((2, 17), (5, 16)), n_mix=1, kernel=K["ln"])
    CASES[f"embed-C{C}"] = Case("embed", C, ((0, 3), (4, 2)), kernel=K["embed"])
    CASES[f"out-C{C}"] = Case("out", C, ((1, 3), (0, 2)), kernel=K["out"])
for C in (128, 256, 2560, 3968, 4096):
    for Dm in (32, 64):
        CASES[f"pre6-C{C}-Dm{Dm}"] = Case("pre6", C, ((2, 3), (0, 1), (7, 4)), n_mix=1, Dm=Dm, kernel=K["pre6"])
        CASES[f"pre6-C{C}-Dm{Dm}-split"] = Case("pre6", C, ((2, 3), (0, 1), (7, 4)), n_mix=1, Dm=Dm, precision=1, kernel=K["pre6"])
# token counts: the cluster kernels and the front half at 1, 2, 15, 16; ln_mix_kernel at every bucket edge above 16
for T in (1, 2, 15, 16):
    CASES[f"cluster-T{T}"] = Case("ln", 1024, ((4, T),), kernel=K["cl"])
    CASES[f"pre6-T{T}"] = Case("pre6", 2048, ((4, T),), n_mix=1, kernel=K["pre6"])
    CASES[f"pre6-T{T}-ones"] = Case("pre6", 2048, tuple((s, 1) for s in range(T)), n_mix=1, kernel=K["pre6"])
for T in (17, 32, 33, 64, 65, 128):
    CASES[f"mix-T{T}"] = Case("ln", 512, ((1, T),), kernel=K["ln"])
    CASES[f"mix-T{T}-ragged"] = Case("ln", 512, ((1, T - T // 2), (0, 1), (3, T // 2 - 1)) if T > 17 else ((1, 9), (0, 8)), kernel=K["ln"])
# entries: many slots of one token, ragged, sparse permuted ids in a pool of 1024
CASES["cluster-many_slots"] = Case("ln", 2048, tuple((s, 1) for s in (5, 0, 9, 2, 7, 11, 1, 3)), kernel=K["cl"])
CASES["cluster-sparse"] = Case("ln", 2048, ((900, 2), (17, 1), (513, 5), (2, 3)), S=1024, kernel=K["cl"])
CASES["mix-sparse"] = Case("ln", 2048, ((900, 20), (17, 1), (513, 5), (2, 30)), S=1024, kernel=K["ln"])
CASES["pre6-sparse"] = Case("pre6", 2560, ((1023, 2), (17, 1), (513, 5)), S=1024, n_mix=1, kernel=K["pre6"])
# residual shapes (n_parts, n_gate): in place, single GPU, and the tensor-parallel shapes (6, 2), (8, 8), (8, 4)
for P, G in ((1, 1), (4, 0), (5, 1), (6, 2), (8, 8), (8, 4)):
    CASES[f"cluster-res{P}_{G}"] = Case("ln", 2048, ((3, 4), (0, 1)), n_parts=P, n_gate=G, kernel=K["cl"])
    CASES[f"mix-res{P}_{G}"] = Case("ln", 2048, ((3, 14), (0, 6)), n_parts=P, n_gate=G, kernel=K["ln"])
    CASES[f"pre6-res{P}_{G}"] = Case("pre6", 2048, ((3, 4), (0, 1)), n_parts=P, n_gate=G, n_mix=1, kernel=K["pre6"])
    CASES[f"out-res{P}_{G}"] = Case("out", 2048, ((3, 4), (0, 1)), n_parts=P, n_gate=G, kernel=K["out"])
    CASES[f"out-res{P}_{G}-T40"] = Case("out", 2048, ((3, 24), (0, 16)), n_parts=P, n_gate=G, options=(capi.OPTION_FULL,) * 2,
                                        kernel=K["out"])
CASES["cluster-in_place"] = Case("ln", 2048, ((3, 4), (0, 1)), n_parts=0, n_gate=0, commit=False, hidden=False, in_place=True,
                                 kernel=K["cl"])
CASES["mix-in_place"] = Case("ln", 2048, ((3, 24), (0, 1)), n_parts=0, n_gate=0, commit=False, hidden=False, in_place=True,
                             kernel=K["ln"])
CASES["pre6-in_place"] = Case("pre6", 2048, ((3, 4), (0, 1)), n_parts=0, n_gate=0, n_mix=1, commit=False, hidden=False,
                              in_place=True, kernel=K["pre6"])
CASES["cluster-no_commit_no_hidden"] = Case("ln", 1024, ((3, 4), (0, 1)), commit=False, hidden=False, kernel=K["cl"])
CASES["out-no_hidden"] = Case("out", 1024, ((3, 4), (0, 1)), hidden=False, commit=False, kernel=K["out"])
# mixes
for m in (1, 2, 4, 6):
    CASES[f"cluster-mix{m}"] = Case("ln", 2560, ((3, 2), (0, 1)), n_mix=m, kernel=K["cl"])
    CASES[f"cluster-mix{m}-split"] = Case("ln", 2560, ((3, 2), (0, 1)), n_mix=m, precision=1, kernel=K["cl"])
    CASES[f"mix-mix{m}"] = Case("ln", 2560, ((3, 20), (0, 1)), n_mix=m, kernel=K["ln"])
# the engine's own configurations
CASES["7B-LN1-pre6"] = Case("pre6", 4096, tuple((s, 1) for s in range(16)), n_parts=1, n_gate=1, n_mix=1, Dm=64, kernel=K["pre6"])
CASES["7B-LN1-pre6-split"] = Case("pre6", 4096, tuple((s, 1) for s in range(16)), n_mix=1, Dm=64, precision=1, kernel=K["pre6"])
CASES["7B-LN2"] = Case("ln", 4096, tuple((s, 1) for s in range(16)), n_parts=1, n_gate=0, n_mix=2, kernel=K["cl"])
CASES["3B-pre6-batch1"] = Case("pre6", 2560, ((0, 1),), n_parts=5, n_gate=1, n_mix=1, Dm=32, kernel=K["pre6"])
CASES["3B-pre6-batch1-split"] = Case("pre6", 2560, ((0, 1),), n_parts=5, n_gate=1, n_mix=1, Dm=32, precision=1, kernel=K["pre6"])
CASES["v7-2.9B-LN1"] = Case("ln", 2560, tuple((s, 1) for s in (4, 1, 6, 0, 7, 2, 5, 3)), n_parts=5, n_gate=0, n_mix=6,
                            kernel=K["cl"])
CASES["out-options"] = Case("out", 2048, ((4, 3), (1, 5), (0, 2), (6, 1)),
                            options=(capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_LAST), kernel=K["out"])
CASES["out-options-split"] = Case("out", 2048, ((4, 3), (1, 5), (0, 2), (6, 1)), precision=1,
                                  options=(capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_LAST), kernel=K["out"])
CASES["out-none"] = Case("out", 1024, ((4, 3), (1, 5)), options=(capi.OPTION_NONE,) * 2, kernel=K["out"])
CASES["prefill-16x8"] = Case("ln", 2048, tuple((s, 8) for s in range(16)), n_parts=4, n_gate=1, n_mix=4, kernel=K["ln"])
CASES["prefill-16x8-out"] = Case("out", 2048, tuple((s, 8) for s in range(16)), n_parts=4, kernel=K["out"])
# data edges
for e in ("const", "big", "slices", "w0", "sat"):
    CASES[f"cluster-{e}"] = Case("ln", 2048, ((3, 4), (0, 1)), edge=e, n_mix=2, kernel=K["cl"])
    CASES[f"mix-{e}"] = Case("ln", 2048, ((3, 14), (0, 6)), edge=e, n_mix=2, kernel=K["ln"])
    CASES[f"pre6-{e}"] = Case("pre6", 2048, ((3, 4), (0, 1)), edge=e, n_mix=1, kernel=K["pre6"])
    CASES[f"out-{e}"] = Case("out", 2048, ((3, 4), (0, 1)), edge=e, options=(capi.OPTION_FULL,) * 2, kernel=K["out"])
CASES["cluster-sat-split"] = Case("ln", 2048, ((3, 4), (0, 1)), edge="sat", precision=1, kernel=K["cl"])
CASES["pre6-sat-split"] = Case("pre6", 2048, ((3, 4), (0, 1)), edge="sat", n_mix=1, precision=1, kernel=K["pre6"])
CASES["embed-ends"] = Case("embed", 1024, ((0, 4), (2, 3)), edge="embed_ends", kernel=K["embed"])
CASES["embed-T128"] = Case("embed", 1024, ((0, 64), (2, 64)), kernel=K["embed"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_ln_stage(name):
    run_case(name, CASES[name])


# ---- launches back to back, positions, and kernels that must agree ------------------------------------------------------
RELAUNCH = {
    "pre6": Case("pre6", 2048, ((3, 4), (0, 1), (5, 2)), n_parts=2, n_mix=1, kernel=K["pre6"]),
    "pre6-split": Case("pre6", 2048, ((3, 4), (0, 1)), n_mix=1, precision=1, kernel=K["pre6"]),
    "cluster": Case("ln", 1088, ((3, 4), (0, 1)), n_mix=3, kernel=K["cl"]),
    "mix": Case("ln", 1088, ((3, 30), (0, 1)), n_mix=3, kernel=K["ln"]),
    "out": Case("out", 1088, ((3, 4), (0, 1)), options=(capi.OPTION_FULL, capi.OPTION_LAST), kernel=K["out"]),
    "embed": Case("embed", 1088, ((3, 4), (0, 1)), kernel=K["embed"]),
}
OUTS = ("x_out", "xx_out", "sx_out", "mix_out", "lora_out", "out5", "head_out", "hidden")


@pytest.mark.parametrize("name", sorted(RELAUNCH))
def test_three_launches_a_b_a(name):
    """Three launches back to back on inputs A, B, A: each slice matches its reference and slices 0 and 2 are identical."""
    _, o, _ = run_case(f"relaunch-{name}", RELAUNCH[name], variants=(0, 1, 0))
    for k in OUTS:
        if o.get(k) is not None:
            a = o[k].view(np.uint16 if o[k].dtype == np.uint16 else np.uint32)
            assert np.array_equal(a[0], a[2]), f"{name}: {k} of launches 0 and 2 differ"
            assert not np.array_equal(a[0], a[1]), f"{name}: {k} of launches 0 and 1 agree"


def entry_out(c: Case, o, slot, k):
    """Rows of output k that belong to the entry of pool slot `slot` (token rows; both split halves)."""
    t0 = 0
    for s, n in c.entries:
        if s == slot:
            break
        t0 += n
    arr = o[k][0]
    if k in ("mix_out", "lora_out", "out5"):
        idx = list(range(t0, t0 + n)) + ([16 + t for t in range(t0, t0 + n)] if c.precision else [])
        return arr[:, idx].view(np.uint16)
    return arr[t0:t0 + n].view(np.uint32)


POSITION = {
    "cluster": (Case("ln", 2048, ((5, 3), (9, 1)), n_mix=2, n_parts=8, n_gate=4),
                Case("ln", 2048, ((2, 2), (9, 1), (7, 6), (5, 3)), n_mix=2, n_parts=8, n_gate=4)),
    "mix": (Case("ln", 2048, ((5, 20), (9, 1)), n_mix=2, n_parts=8, n_gate=4),
            Case("ln", 2048, ((2, 40), (9, 1), (7, 6), (5, 20)), n_mix=2, n_parts=8, n_gate=4)),
    "pre6": (Case("pre6", 2048, ((5, 3), (9, 1)), n_mix=1, n_parts=6, n_gate=2),
             Case("pre6", 2048, ((2, 2), (9, 1), (7, 6), (5, 3)), n_mix=1, n_parts=6, n_gate=2)),
    "pre6-split": (Case("pre6", 2048, ((5, 3), (9, 1)), n_mix=1, precision=1),
                   Case("pre6", 2048, ((2, 2), (9, 1), (7, 6), (5, 3)), n_mix=1, precision=1)),
    "out": (Case("out", 2048, ((5, 3), (9, 1)), options=(capi.OPTION_FULL,) * 2),
            Case("out", 2048, ((2, 2), (9, 1), (7, 6), (5, 3)), options=(capi.OPTION_FULL,) * 4)),
    "embed": (Case("embed", 2048, ((5, 3), (9, 1))), Case("embed", 2048, ((2, 2), (9, 1), (7, 6), (5, 3)))),
}


@pytest.mark.parametrize("name", sorted(POSITION))
def test_entry_rows_do_not_depend_on_position(name):
    """The same entry (same per-token inputs) placed at another position among other companions gives identical rows."""
    a, b = POSITION[name]
    _, oa, ka = run_case(f"position-{name}-a", a)
    _, ob, kb = run_case(f"position-{name}-b", b)
    assert ka == kb
    for k in OUTS:
        if oa.get(k) is None:
            continue
        if k == "head_out":         # every token produces a row: the entry's rows are its token rows
            k2 = oa[k][0][:3], ob[k][0][2 + 1 + 6:2 + 1 + 6 + 3]
            assert np.array_equal(*k2), f"{name}: head rows moved with the entry"
            continue
        assert np.array_equal(entry_out(a, oa, 5, k), entry_out(b, ob, 5, k)), f"{name}: {k} depends on the entry's position"


def test_pre6_phase1_equals_the_cluster_ln_kernel():
    """pre6_kernel and ln_mix_cluster_kernel both run pre_ln_slice: the same single-mix LN gives identical rows."""
    for prec in (0, 1):
        c6 = Case("pre6", 2560, ((3, 4), (0, 1), (8, 7)), n_parts=6, n_gate=2, n_mix=1, precision=prec, kernel=K["pre6"])
        cl = dataclasses.replace(c6, stage="ln", kernel=K["cl"])
        _, o6, _ = run_case(f"phase1-pre6-p{prec}", c6)
        _, ol, _ = run_case(f"phase1-cluster-p{prec}", cl)
        for k in ("x_out", "xx_out", "sx_out", "hidden"):
            assert np.array_equal(o6[k].view(np.uint32), ol[k].view(np.uint32)), f"precision {prec}: {k}"
        assert np.array_equal(o6["mix_out"], ol["mix_out"]), f"precision {prec}: mix 0"
        assert np.array_equal(o6["commit_dst"].view(np.uint32), ol["commit_dst"].view(np.uint32))


@pytest.mark.parametrize("parts", [(1, 1), (5, 1), (8, 8), (8, 4), (6, 2), (4, 0)])
def test_residual_row_equals_residual_vec(parts):
    """pre6.cuh's residual_vec is the same arithmetic as mix.cuh's residual_row: for the same token, ln_mix_kernel (T > 16)
    and the cluster kernels write identical x_out rows."""
    P, G = parts
    big = Case("ln", 2048, ((3, 4), (7, 20)), n_parts=P, n_gate=G, kernel=K["ln"])
    small = Case("ln", 2048, ((3, 4),), n_parts=P, n_gate=G, kernel=K["cl"])
    six = Case("pre6", 2048, ((3, 4),), n_parts=P, n_gate=G, n_mix=1, kernel=K["pre6"])
    _, ob, _ = run_case(f"resid-mix-{P}_{G}", big)
    _, os_, _ = run_case(f"resid-cluster-{P}_{G}", small)
    _, o6, _ = run_case(f"resid-pre6-{P}_{G}", six)
    row = ob["x_out"][0, :4].view(np.uint32)
    assert np.array_equal(row, os_["x_out"][0].view(np.uint32))
    assert np.array_equal(row, o6["x_out"][0].view(np.uint32))
