"""The snapshot variants of the step kernels driven alone through b200rwkv_op_wkv / b200rwkv_op_ln with snapshot arguments:
the step's snapshot block comes from the engine's own fill_snap (as b200rwkv_infer_snapshots builds it), and the launch runs
with the step shape's snap / MTX set, so wkv_kernel<..., SNAP = true>, the records of the LN stages and ln_out's snapshot
head rows run exactly as in a snapshot step.

Each case runs the same inputs twice, once plain and once with snapshots, and checks bit for bit:
  * every output the plain launch writes is unchanged by the snapshots;
  * WKV: the record of token p of an entry equals the state a plain launch of that entry's first p tokens leaves from the
    same initial state.  tests/test_gpu_wkv.py holds such cut runs bit-identical across the staged, per-token and fold
    paths and holds each of them to a float64 reference, so every record is tied to that reference;
  * LN stages: the record equals commit_src's row of its token when the stage commits, and is left alone when it does not
    (layer 0's LN1 in a step);
  * ln_out: row k of snap_head_out equals the head row the same token gets when its entry is FULL (the same LN result
    through the same store), for the k-th snapshot token without a head row;
  * record cells outside [snap_off, snap_off + part) and snap_head_out rows nobody owns keep their NaN sentinels.
"""
import dataclasses
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi

import test_gpu_ln as LN
import test_gpu_wkv as W

pytestmark = pytest.mark.gpu

SENT32, SENT16 = W.SENT32, W.SENT16
OFF = 12                            # snap_off: the record part starts past a few sentinel cells ...
TAIL = 20                           # ... and ends before a few more


def u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def starts(entries):
    return np.cumsum([0] + [n for _, n in entries])[:-1]


# ---- WKV ---------------------------------------------------------------------------------------------------------------
def wkv_case(name, c: W.Case, at):
    """`at`: {entry index: positions 1..n}.  Returns the worst record / plain difference (0 when bit-identical)."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    H, C, S = c.H, c.H * 64, c.pool
    T = sum(n for _, n in c.entries)
    layer = c.layer
    vf = W.f32(rng.standard_normal((T, C))) if c.version == 7 and layer else None
    ch, tok = W.make_inputs(c, rng, layer, vf)
    state0 = W.sentinel32((S, H, 64, 64))
    for s, _ in c.entries:
        state0[s] = W.f32(rng.standard_normal((H, 64, 64)) * 0.3)
    t0 = starts(c.entries)
    snaps = [(e, p) for e, ps in at.items() for p in ps]
    snap_tok = [int(t0[e]) + p - 1 for e, p in snaps]
    order = rng.permutation(len(snaps))             # the records in another order than the tokens
    snaps, snap_tok = [snaps[i] for i in order], [snap_tok[i] for i in order]

    runs = []
    for with_snap in (False, True):
        st = state0.copy()
        tk = {k: v.copy() for k, v in tok.items()}
        kw = {}
        if with_snap:
            rec = W.sentinel32((len(snaps), OFF + H * 4096 + TAIL))
            kw = dict(snap_tok=snap_tok, snap_rec=rec, snap_off=OFF)
        out = W.launch(c, ch, tk, st, layer, **kw)
        runs.append((out, st, tk.get("v_first"), kw.get("snap_rec")))
    (out_p, st_p, vf_p, _), (out_s, st_s, vf_s, rec) = runs
    assert np.array_equal(out_p, out_s), f"{name}: out changed by the snapshots"
    assert np.array_equal(u32(st_p), u32(st_s)), f"{name}: state changed by the snapshots"
    if c.version == 7:
        assert np.array_equal(u32(vf_p), u32(vf_s)), f"{name}: v_first changed by the snapshots"
    assert np.all(u32(rec[:, :OFF]) == SENT32) and np.all(u32(rec[:, OFF + H * 4096:]) == SENT32), \
        f"{name}: a record cell outside the WKV part was written"

    worst = 0.0
    for k, (e, p) in enumerate(snaps):
        slot, n = c.entries[e]
        cut = dataclasses.replace(c, entries=((slot, p),), S=S)
        tk = {key: v[t0[e]:t0[e] + p].copy() for key, v in tok.items()}
        st = state0.copy()
        W.launch(cut, ch, tk, st, layer)
        want = st[slot].reshape(-1)
        got = rec[k, OFF:OFF + H * 4096]
        d = np.abs(got.astype(np.float64) - want)
        worst = max(worst, float(np.nanmax(np.where(np.isnan(d), np.inf, d))))
        assert np.array_equal(u32(got), u32(want)), f"{name}: record of entry {e} position {p} != the state after p tokens"
    return worst


WKV_CASES = {}
STAGED = ((0, 1), (1, 2), (2, 4), (3, 3))          # staged runs (<= 4 tokens), a snapshot at every token
EVERY = {e: list(range(1, n + 1)) for e, (_, n) in enumerate(STAGED)}
for vn, vk in W.VERSIONS.items():
    WKV_CASES[f"{vn}-staged_every"] = (W.Case(entries=STAGED, **vk), EVERY)
    WKV_CASES[f"{vn}-staged_every_split"] = (W.Case(entries=STAGED, precision=1, **vk), EVERY)
    # per-token runs (the v6 fold versions: the per-token fold), snapshots at 1, the middle and the end
    for n in (5, 17, 65, 128):
        WKV_CASES[f"{vn}-run{n}"] = (W.Case(entries=((1, n),), H=2, **vk), {0: sorted({1, (n + 1) // 2, n})})
    WKV_CASES[f"{vn}-run5_split"] = (W.Case(entries=((1, 5),), H=2, precision=1, **vk), {0: [1, 3, 5]})
    # ragged batches, some entries without a snapshot
    WKV_CASES[f"{vn}-ragged"] = (W.Case(entries=((0, 5), (1, 1), (2, 4), (3, 7), (4, 3)), **vk), {0: [2, 5], 2: [1, 4], 3: [7]})
    WKV_CASES[f"{vn}-ragged_split"] = (W.Case(entries=((1, 5), (3, 4), (0, 7)), precision=1, **vk), {0: [5], 2: [1, 3, 7]})
for prec in (0, 1):
    WKV_CASES[f"v6fold128-7b_decode16{'_split' if prec else ''}"] = (
        W.Case(version=6, Dd=128, H=64, entries=tuple((s, 1) for s in range(16)), precision=prec),
        {e: [1] for e in range(0, 16, 3)})


@pytest.mark.parametrize("name", list(WKV_CASES))
def test_wkv_snapshot_records(name):
    c, at = WKV_CASES[name]
    worst = wkv_case(name, c, at)
    print(f"\n[snap-wkv] {name}: {sum(len(v) for v in at.values())} records, worst |record - state| {worst:.3g}")


# ---- LN stages -----------------------------------------------------------------------------------------------------------
def ln_snap_run(c: LN.Case, x, snap_tok, head_rows=0):
    rec = W.sentinel32((len(snap_tok), OFF + c.C + TAIL))
    kw = dict(snap_tok=snap_tok, snap_rec=rec, snap_off=OFF)
    if c.stage == "out":
        kw["snap_head_out"] = np.full((head_rows, c.C), SENT16, np.uint16)
    o, kern, _ = LN.run_op(c, x, 1, **kw)
    return o, kern, rec, kw.get("snap_head_out")


def assert_outputs_equal(name, o_p, o_s):
    for k in LN.OUTS + ("commit_dst", "x_in_after"):
        if o_p.get(k) is not None:
            assert np.array_equal(np.ascontiguousarray(o_p[k]).view(np.uint8), np.ascontiguousarray(o_s[k]).view(np.uint8)), \
                f"{name}: {k} changed by the snapshots"


def check_records(name, c: LN.Case, x, rec, snap_tok):
    C = c.C
    assert np.all(u32(rec[:, :OFF]) == SENT32) and np.all(u32(rec[:, OFF + C:]) == SENT32), \
        f"{name}: a record cell outside the shift row was written"
    part = rec[:, OFF:OFF + C]
    if c.commit:
        want = x["commit_src"][0][snap_tok]
        bad = np.nonzero(np.any(u32(part) != u32(want), axis=1))[0]
        assert bad.size == 0, f"{name}: records of tokens {[snap_tok[i] for i in bad]} != commit_src " \
                              f"(first bad column {int(np.argmax(u32(part[bad[0]]) != u32(want[bad[0]])))})"
    else:
        assert np.all(u32(part) == SENT32), f"{name}: a stage without a commit wrote a record"


def ln_case(name, c: LN.Case, snap_tok):
    x = LN.make_inputs(c, (0,))
    o_p, k_p, _ = LN.run_op(c, x, 1)
    o_s, k_s, rec, _ = ln_snap_run(c, x, snap_tok)
    assert k_p == k_s and (c.kernel < 0 or k_s[0] == c.kernel), f"{name}: kernels {k_p} / {k_s}"
    assert_outputs_equal(name, o_p, o_s)
    check_records(name, c, x, rec, snap_tok)
    print(f"\n[snap-ln] {name} kernel {k_s}: {len(snap_tok)} records of {c.T} tokens, commit {c.commit}")


K = LN.K
LN_CASES = {
    "mix-T21": (LN.Case("ln", 512, ((1, 9), (0, 12)), kernel=K["ln"]), [0, 4, 8, 9, 20]),
    "mix-T40-res8_4": (LN.Case("ln", 2048, ((3, 24), (5, 16)), n_parts=8, n_gate=4, n_mix=4, kernel=K["ln"]), [23, 0, 39, 24, 10]),
    "mix-T128-C4160": (LN.Case("ln", 4160, ((2, 100), (0, 28)), n_mix=1, kernel=K["ln"]), list(range(0, 128, 7)) + [127]),
    "mix-no_commit": (LN.Case("ln", 1024, ((3, 24), (0, 1)), commit=False, kernel=K["ln"]), [0, 5, 24]),
    "mix-in_place_no_commit": (LN.Case("ln", 2048, ((3, 24), (0, 1)), n_parts=0, n_gate=0, commit=False, hidden=False,
                                       in_place=True, kernel=K["ln"]), [1, 24]),
}
for C in (1024, 1088, 2048, 4096, 4160):
    LN_CASES[f"cluster-C{C}"] = (LN.Case("ln", C, ((3, 5), (0, 1), (9, 9)), kernel=K["cl"]), [0, 2, 4, 5, 6, 14])
    LN_CASES[f"cluster-C{C}-split"] = (LN.Case("ln", C, ((3, 5), (0, 1), (9, 4)), precision=1, kernel=K["cl"]), [4, 5, 0, 9])
LN_CASES["cluster-v7-2.9B-LN1"] = (LN.Case("ln", 2560, tuple((s, 1) for s in (4, 1, 6, 0, 7, 2, 5, 3)), n_parts=5, n_gate=0,
                                           n_mix=6, kernel=K["cl"]), list(range(8)))
LN_CASES["cluster-no_commit"] = (LN.Case("ln", 1088, ((3, 5), (0, 1)), commit=False, kernel=K["cl"]), [0, 4, 5])
LN_CASES["cluster-in_place_no_commit"] = (LN.Case("ln", 2048, ((3, 4), (0, 1)), n_parts=0, n_gate=0, commit=False, hidden=False,
                                                  in_place=True, kernel=K["cl"]), [3, 4])
for Dm in (32, 64):
    for prec in (0, 1):
        sfx = f"-Dm{Dm}" + ("-split" if prec else "")
        LN_CASES["pre6-C2560" + sfx] = (LN.Case("pre6", 2560, ((2, 3), (0, 1), (7, 4)), n_mix=1, Dm=Dm, precision=prec,
                                                kernel=K["pre6"]), [0, 1, 2, 3, 6, 7])
    LN_CASES[f"pre6-7B-LN1-Dm{Dm}"] = (LN.Case("pre6", 4096, tuple((s, 1) for s in range(16)), n_mix=1, Dm=Dm, kernel=K["pre6"]),
                                       list(range(0, 16, 2)))
LN_CASES["pre6-no_commit"] = (LN.Case("pre6", 2048, ((3, 4), (0, 1)), commit=False, n_mix=1, kernel=K["pre6"]), [0, 3, 4])
LN_CASES["pre6-in_place_no_commit"] = (LN.Case("pre6", 2048, ((3, 4), (0, 1)), n_parts=0, n_gate=0, n_mix=1, commit=False,
                                               hidden=False, in_place=True, kernel=K["pre6"]), [0, 4])


@pytest.mark.parametrize("name", list(LN_CASES))
def test_ln_snapshot_records(name):
    c, snap_tok = LN_CASES[name]
    ln_case(name, c, snap_tok)


# ---- ln_out: records and the snapshot head rows ---------------------------------------------------------------------------
NONE, LAST, FULL = capi.OPTION_NONE, capi.OPTION_LAST, capi.OPTION_FULL


def out_case(X, precision=0, C=1024):
    """An ln_out step with X snapshot tokens that have no head row: a NONE entry with a snapshot at every token, a LAST entry
    with snapshots mid-run and at its end (which has a head row), a FULL entry with one."""
    if X == 128 or (precision and X == 16):
        entries, options, snaps = ((5, X),), (NONE,), list(range(X))
    elif X == 1:
        entries, options, snaps = ((5, 3),), (LAST,), [0, 2]
    else:
        n = X - 1
        entries, options = ((5, n), (2, 3), (7, 2)), (NONE, LAST, FULL)
        snaps = list(range(n)) + [n, n + 2, n + 4]
    c = LN.Case("out", C, entries, options=options, precision=precision, kernel=K["out"])
    return c, snaps


def mt(rows):
    return 1 if rows <= 16 else 2 if rows <= 32 else 4 if rows <= 64 else 8


def ln_out_case(name, c: LN.Case, snaps):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    snap_tok = [snaps[i] for i in rng.permutation(len(snaps))]
    split = c.precision == 1
    outrow = []
    for (_, n), op in zip(c.entries, c.options):
        outrow += [op == FULL or (op == LAST and j == n - 1) for j in range(n)]
    xtok = [t for t in snap_tok if not outrow[t]]          # row k of snap_head_out: the k-th of snap_tok without a head row
    X = len(xtok)
    rows_x = 32 if split else 16 * mt(X)
    x = LN.make_inputs(c, (0,))
    o_p, k_p, _ = LN.run_op(c, x, 1)
    o_s, k_s, rec, sho = ln_snap_run(c, x, snap_tok, rows_x)
    assert k_p == k_s == (K["out"], k_p[1], c.precision), f"{name}: kernels {k_p} / {k_s}"
    assert_outputs_equal(name, o_p, o_s)
    check_records(name, c, x, rec, snap_tok)
    # the head rows every token gets when its entry is FULL
    full = dataclasses.replace(c, options=(FULL,) * len(c.entries))
    o_f, _, _ = LN.run_op(full, x, 1)
    head = o_f["head_out"][0]
    own = list(range(X)) + (list(range(16, 16 + X)) if split else [])
    for k, t in enumerate(xtok):
        assert np.array_equal(sho[k], head[t]), f"{name}: snapshot head row {k} != the FULL head row of token {t}"
        if split:
            assert np.array_equal(sho[16 + k], head[16 + t]), f"{name}: lo half of snapshot head row {k} (token {t})"
    keep = np.ones(rows_x, bool)
    keep[own] = False
    assert np.all(sho[keep] == SENT16), f"{name}: a snapshot head row past the X = {X} rows was written"
    print(f"\n[snap-ln_out] {name}: X {X} rows_x {rows_x}, {len(snap_tok) - X} snapshot tokens with a head row")


OUT_CASES = {f"X{X}": out_case(X) for X in (1, 15, 16, 17, 32, 33, 64, 65, 128)}
OUT_CASES.update({f"X{X}-split": out_case(X, precision=1) for X in (1, 11, 16)})
OUT_CASES["X40-C4160"] = out_case(40, C=4160)
OUT_CASES["X7-C8192"] = out_case(7, C=8192)


@pytest.mark.parametrize("name", list(OUT_CASES))
def test_ln_out_snapshot_rows(name):
    c, snaps = OUT_CASES[name]
    ln_out_case(name, c, snaps)
