"""Snapshots inside one infer call (b200rwkv_infer_snapshots): the state of a slot after a chosen token of its entry, with
that token's logits row, taken by the step's own kernels.  Checked against the NumPy oracle after the same tokens
(1e-3 relative, same argmax), against state_read / logits_out bit for bit where they hold the same thing, and for leaving
every other output of the call bit-identical to infer_ex."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

from adapter_oracle import AdapterOracle

pytestmark = pytest.mark.gpu

LAST, FULL, NONE, SCORE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_SCORE


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(preset, max_batch=4, chunk=32, **kw):
        key = (preset if isinstance(preset, str) else repr(preset), max_batch, chunk, tuple(sorted(kw.items())))
        if key not in cache:
            st = synth.make_st(preset, 0)
            cache[key] = (runtime.Model(st, max_batch=max_batch, token_chunk_size=chunk, **kw), st)
        return cache[key]

    yield get
    for m, _ in cache.values():
        m.close()


@pytest.fixture(scope="module")
def ad_model():
    """tiny6 with one unblended adapter (pairs on att.key / att.value / ffn.key and the head), the even slots bound; steps of
    at most 16 tokens, so every step is decode-shaped."""
    st = synth.make_st("tiny6", 0)
    ad = synth.make_lora_st("tiny6", rank=8, seed=11, targets=("att.key", "att.value", "ffn.key"))
    m = runtime.Model(st, max_batch=16, token_chunk_size=16, adapters=[(ad, 0.75)])
    m.bind_adapter(list(range(0, 16, 2)), [1] * 8)
    yield m, st, ad
    m.close()


def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def toks_for(n, seed, V):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, n)]


def reset(m, slots):
    for s in slots:
        m.state.load(m.state.init(), s)


def check_snapshot(m, orc, snap, tokens, p, tol=1e-3):
    st, row = m.state.snapshot_back(snap, with_logits=True)
    want_row, want_st = orc.run(tokens[:p], orc.state_init())
    assert rel(st, want_st) <= tol, (p, rel(st, want_st))
    assert rel(row, want_row[0]) <= tol and int(row.argmax()) == int(want_row[0].argmax()), (p, rel(row, want_row[0]))


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
@pytest.mark.parametrize("chunk", [32, 128])
def test_snapshot_content_against_oracle(models, preset, chunk):
    m, st = models(preset, chunk=chunk)
    orc = O.Oracle(O.parse_st(st), "f16")
    V = m.info["num_vocab"]
    for n, opt in ((45, LAST), (130, NONE), (300, FULL)):
        reset(m, [0])
        toks = toks_for(n, n, V)
        # position 1, mid-step, the last token of an internal step, the first of the next one, the entry's last token
        at = sorted({1, chunk // 2, chunk, chunk + 1, n} & set(range(1, n + 1)))
        _, _, snaps = m.infer_snapshots([0], [n], toks, [opt], [(0, p) for p in at])
        for p, s in zip(at, snaps):
            check_snapshot(m, orc, s, toks, p)
            s.free()


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_ragged_mixed_options(models, preset):
    m, st = models(preset, max_batch=4, chunk=32)
    orc = O.Oracle(O.parse_st(st), "f16")
    V = m.info["num_vocab"]
    ntok, opts = [40, 7, 33, 12], [LAST, FULL, NONE, SCORE]
    toks = [toks_for(n, 100 + i, V) for i, n in enumerate(ntok)]
    at = [(0, 1), (0, 20), (0, 40), (1, 3), (1, 7), (2, 16), (2, 33), (3, 1), (3, 12)]
    reset(m, [3, 1, 0, 2])
    slots = [3, 1, 0, 2]
    _, _, snaps = m.infer_snapshots(slots, ntok, [x for t in toks for x in t], opts, at)
    for (e, p), s in zip(at, snaps):
        check_snapshot(m, orc, s, toks[e], p)
        s.free()


def run_pair(m, slots, ntok, flat, opts, at, pool=False):
    """The same call through infer_ex and infer_snapshots from the same states (kept rows included: each slot's state and
    kept row are put back from a snapshot of them): every output of both.  `pool`: pooled hidden rows on, or off."""
    init = [m.state.read(s) for s in slots]
    outs = []
    for use_snap in (False, True):
        for s, x in zip(slots, init):
            m.state.write(x, s)
        m.keep_hidden_pooled([0], "mean") if pool else m.keep_hidden_pooled([])
        n0 = m.launch_count()
        if use_snap:
            rows, scores, snaps = m.infer_snapshots(slots, ntok, flat, opts, at)
        else:
            rows, scores = m.infer_ex(slots, ntok, flat, opts)
            snaps = []
        launches = m.launch_count() - n0
        states = [m.state.back(s) for s in slots]
        kept = []
        for i, s in enumerate(slots):
            t = m.state.read(s)
            kept.append(m.state.snapshot_back(t, with_logits=True)[1] if opts[i] != NONE and ntok[i] else None)
            t.free()
        pooled = m.last_hidden_pooled(0)[0] if pool else None
        outs.append((rows, scores, states, kept, pooled, launches, snaps))
    for x in init:
        x.free()
    m.keep_hidden_pooled([])
    return outs


def assert_same(a, b):
    for x, y in zip(a[0], b[0]):
        assert np.array_equal(x, y)
    for x, y in zip(a[1], b[1]):
        assert (x is None) == (y is None)
        if x is not None:
            assert np.array_equal(x[0], y[0], equal_nan=True) and np.array_equal(x[1], y[1])
    for x, y in zip(a[2], b[2]):
        assert np.array_equal(x, y)
    for x, y in zip(a[3], b[3]):
        assert (x is None) == (y is None) and (x is None or np.array_equal(x, y))
    if a[4] is not None:
        assert np.array_equal(a[4], b[4])


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_bit_identity_with_infer_ex(models, preset):
    m, _ = models(preset, max_batch=4, chunk=32)
    V = m.info["num_vocab"]
    slots, ntok, opts = [2, 0, 1], [50, 9, 4], [FULL, NONE, SCORE]
    flat = toks_for(sum(ntok), 7, V)
    at = [(0, 1), (0, 33), (0, 50), (1, 5), (1, 9), (2, 2)]
    reset(m, slots)
    for pool in (False, True, False):          # before, with and after pooled hidden rows (turned off again)
        plain, snap = run_pair(m, slots, ntok, flat, opts, at, pool)
        assert_same(plain, snap)
        # a FULL snapshot carries exactly its logits_out row; an end-of-entry one equals state_read after the call
        _, row = m.state.snapshot_back(snap[6][2], with_logits=True)
        assert np.array_equal(row, snap[0][0][49])
        st_end, row_end = m.state.snapshot_back(snap[6][2], with_logits=True)
        rd = m.state.read(2)
        st_rd, row_rd = m.state.snapshot_back(rd, with_logits=True)
        assert np.array_equal(st_end, st_rd) and np.array_equal(row_end, row_rd)
        assert np.array_equal(m.state.snapshot_back(snap[6][4]), snap[2][1])       # NONE entry's end: the state
        rd.free()
        for s in snap[6]:
            s.free()
    # nsnap = 0 launches what infer_ex launches, with the same bits
    plain, none = run_pair(m, slots, ntok, flat, opts, [])
    assert_same(plain, none)
    assert plain[5] == none[5]


def test_score_entry_rows_match_full(models):
    """A SCORE snapshot's row is the row its next token was scored from: the FULL row of the same call."""
    m, _ = models("tiny6", max_batch=4, chunk=32)
    V = m.info["num_vocab"]
    flat = toks_for(6, 3, V)
    reset(m, [0, 1])
    rows, _, snaps = m.infer_snapshots([0, 1], [6, 6], flat + flat, [FULL, SCORE], [(1, p) for p in range(1, 7)])
    for p, s in enumerate(snaps, 1):
        assert np.array_equal(m.state.snapshot_back(s, with_logits=True)[1], rows[0][p - 1])
        s.free()


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_restore_and_continue(models, preset):
    m, st = models(preset, max_batch=2, chunk=32)
    orc = O.Oracle(O.parse_st(st), "f16")
    V = m.info["num_vocab"]
    toks = toks_for(70, 5, V)
    reset(m, [0])
    p = 37
    _, _, (snap,) = m.infer_snapshots([0], [70], toks, [NONE], [(0, p)])
    m.state.write(snap, 1)
    ids, _ = m.sample_topk([1], top_k=1)
    want, _ = orc.run(toks[:p], orc.state_init())
    assert int(ids[0, 0]) == int(want[0].argmax())
    rows = m.infer_raw([1], [70 - p], toks[p:], [LAST])
    want, want_st = orc.run(toks, orc.state_init())
    assert rel(rows[0][0], want[0]) <= 1e-3 and int(rows[0][0].argmax()) == int(want[0].argmax())
    assert rel(m.state.back(1), want_st) <= 1e-3
    snap.free()


def verify_case(m, orc_for, B, V, tol=1e-3):
    """B slots, one SCORE entry of 4 tokens each, snapshots at 1..4 of every entry."""
    slots = list(range(B))
    reset(m, slots)
    toks = [toks_for(4, 40 + s, V) for s in slots]
    at = [(e, p) for e in range(B) for p in range(1, 5)]
    _, scores, snaps = m.infer_snapshots(slots, [4] * B, [x for t in toks for x in t], [SCORE] * B, at)
    for (e, p), s in zip(at, snaps):
        if e in (0, B - 1):
            check_snapshot(m, orc_for(e), s, toks[e], p, tol)
        s.free()


@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7"])
def test_decode_shaped_verify(models, preset, B):
    m, st = models(preset, max_batch=16, chunk=128)
    orc = O.Oracle(O.parse_st(st), "f16")
    verify_case(m, lambda e: orc, B, m.info["num_vocab"])


@pytest.mark.parametrize("B", [1, 16])
def test_decode_verify_precision1(models, B):
    m, st = models("tiny6", max_batch=16, chunk=128, exact=True)
    orc = O.Oracle(O.parse_st(st), "f32")
    verify_case(m, lambda e: orc, B, m.info["num_vocab"])


def test_decode_verify_int8(models):
    m, st = models("tiny6", max_batch=16, chunk=128, quant=2, quant_type="Int8")
    orc = O.Oracle(Q.quantize_model(O.parse_st(st), 2, Q.QUANT_INT8), "f16")
    verify_case(m, lambda e: orc, 16, m.info["num_vocab"])


def test_decode_verify_bound_adapter():
    st = synth.make_st("tiny6", 0)
    ad = synth.make_lora_st("tiny6", rank=8, seed=11, targets=("att.key", "att.value", "ffn.key"))
    m = runtime.Model(st, max_batch=16, token_chunk_size=128, adapters=[(ad, 0.75)])
    try:
        m.bind_adapter(list(range(0, 16, 2)), [1] * 8)
        w = O.parse_st(st)
        base, bound = O.Oracle(w, "f16"), AdapterOracle(w, "f16", (O.parse_st(ad), 0.75))
        verify_case(m, lambda e: bound if e % 2 == 0 else base, 16, m.info["num_vocab"])
        # mid-run NONE snapshots of a bound slot go through the adapter's own head launch
        reset(m, [0])
        toks = toks_for(20, 9, m.info["num_vocab"])
        _, _, snaps = m.infer_snapshots([0], [20], toks, [NONE], [(0, 5), (0, 20)])
        for p, s in zip((5, 20), snaps):
            check_snapshot(m, bound, s, toks, p)
            s.free()
    finally:
        m.close()


def test_decode_verify_7b_layer_shape():
    shp = dataclasses.replace(synth.PRESETS["v6-7b"], L=1, V=4096)
    st = synth.make_st(shp, 0)
    m = runtime.Model(st, max_batch=16, token_chunk_size=128)
    try:
        orc = O.Oracle(O.parse_st(st), "f16")
        verify_case(m, lambda e: orc, 16, 4096)
    finally:
        m.close()


def test_reuse_overwrites_in_place(models):
    m, st = models("tiny6", max_batch=2, chunk=32)
    orc = O.Oracle(O.parse_st(st), "f16")
    V = m.info["num_vocab"]
    reset(m, [0])
    plain = m.state.read(0)          # a snapshot without a row (fresh slot, no kept row)
    t1 = toks_for(8, 1, V)
    _, _, (a, b) = m.infer_snapshots([0], [8], t1, [SCORE], [(0, 2), (0, 8)])
    before = m.state.cache_stats()
    reset(m, [0])
    t2 = toks_for(8, 2, V)
    _, _, (a2, b2, c2) = m.infer_snapshots([0], [8], t2, [NONE], [(0, 3), (0, 6), (0, 8)], reuse=[a, b, plain])
    assert (a2.id, b2.id, c2.id) == (a.id, b.id, plain.id)
    assert m.state.cache_stats()["bytes_used"] >= before["bytes_used"]
    after = m.state.cache_stats()
    check_snapshot(m, orc, a2, t2, 3)
    check_snapshot(m, orc, b2, t2, 6)
    check_snapshot(m, orc, c2, t2, 8)
    # a second reuse changes no byte count
    m.infer_snapshots([0], [8], t2, [NONE], [(0, 3), (0, 6), (0, 8)], reuse=[a, b, plain])
    assert m.state.cache_stats()["bytes_used"] == after["bytes_used"]
    for s in (a, b, plain):
        s.free()


def test_refusals_change_nothing(models):
    m, _ = models("tiny6", max_batch=2, chunk=32)
    V = m.info["num_vocab"]
    reset(m, [0, 1])
    m.infer_raw([0, 1], [3, 3], toks_for(6, 4, V), [LAST, LAST])
    _, _, (keep,) = m.infer_snapshots([0], [2], toks_for(2, 5, V), [LAST], [(0, 1)])
    st0, st1 = m.state.back(0), m.state.back(1)
    k_st, k_row = m.state.snapshot_back(keep, with_logits=True)
    ids0, _ = m.sample_topk([0, 1], top_k=1)
    toks = toks_for(6, 6, V)
    bad = [
        ([(2, 1)], None, capi.ERR_INVALID),             # entry out of range
        ([(0, 0)], None, capi.ERR_INVALID),             # position 0
        ([(0, 4)], None, capi.ERR_INVALID),             # past ntok
        ([(0, 2), (0, 2)], None, capi.ERR_INVALID),     # duplicate (entry, position)
        ([(0, 1), (1, 1)], [keep.id, keep.id], capi.ERR_INVALID),     # one id twice
        ([(0, 1)], [987654321], capi.ERR_STATE),        # unknown id
    ]
    for at, reuse, code in bad:
        with pytest.raises(capi.B200Error) as ex:
            m.infer_snapshots([0, 1], [3, 3], toks, [LAST, FULL], at, reuse=reuse)
        assert ex.value.code == code, (at, ex.value.code)
    args = capi.InferArgs(capi.C.sizeof(capi.InferArgs), 0, None, None, None, None, None, 0, None, None, None)
    assert capi.lib().b200rwkv_infer_snapshots(m._h, capi.C.byref(args), -1, None, None, None) == capi.ERR_INVALID
    assert capi.lib().b200rwkv_infer_snapshots(m._h, capi.C.byref(args), 1, None, None, None) == capi.ERR_INVALID
    assert np.array_equal(m.state.back(0), st0) and np.array_equal(m.state.back(1), st1)
    s2, r2 = m.state.snapshot_back(keep, with_logits=True)
    assert np.array_equal(s2, k_st) and np.array_equal(r2, k_row)
    ids1, _ = m.sample_topk([0, 1], top_k=1)
    assert np.array_equal(ids0, ids1)
    keep.free()


def test_end_of_entry_snapshot_equals_state_read(models):
    """A snapshot at an entry's last token holds what state_read returns after the call, bit for bit: the state for every
    option, and the kept row for LAST / FULL / SCORE entries."""
    m, _ = models("tiny6", max_batch=4, chunk=32)
    V = m.info["num_vocab"]
    slots, ntok, opts = [0, 1, 2, 3], [5, 9, 6, 7], [LAST, FULL, SCORE, NONE]
    reset(m, slots)
    _, _, snaps = m.infer_snapshots(slots, ntok, toks_for(sum(ntok), 8, V), opts, [(i, n) for i, n in enumerate(ntok)])
    for s, o, sn in zip(slots, opts, snaps):
        rd = m.state.read(s)
        st_sn, row_sn = m.state.snapshot_back(sn, with_logits=True)
        assert np.array_equal(st_sn, m.state.snapshot_back(rd)), o
        if o != NONE:
            assert np.array_equal(row_sn, m.state.snapshot_back(rd, with_logits=True)[1]), o
        rd.free()
        sn.free()


def decode_call(V, B=16):
    """B slots of 1 to 4 tokens with mixed options, snapshots at an entry's first token, mid-run and at its end.  On an
    engine with token_chunk_size 16 every step holds at most 16 tokens, so the T <= 16 LN / front-half kernels run, and the
    snapshot head launch runs for the NONE / mid-run LAST tokens."""
    ntok = [1 + s % 4 for s in range(B)]
    opts = [(LAST, FULL, NONE, SCORE)[s % 4] for s in range(B)]
    at = sorted({(e, p) for e in range(B) for p in (1, (ntok[e] + 1) // 2, ntok[e])})
    return list(range(B)), ntok, toks_for(sum(ntok), 21, V), opts, at


@pytest.mark.parametrize("case", ["tiny5", "tiny6", "tiny7", "small6", "tiny6-precision1", "tiny6-adapter"])
def test_bit_identity_decode_shaped(models, ad_model, case):
    if case == "tiny6-adapter":
        m = ad_model[0]
    elif case == "tiny6-precision1":
        m = models("tiny6", max_batch=16, chunk=16, exact=True)[0]
    else:
        m = models(case, max_batch=16, chunk=16)[0]
    V = m.info["num_vocab"]
    slots, ntok, flat, opts, at = decode_call(V)
    reset(m, slots)
    for pool in (False, True, False):
        plain, snap = run_pair(m, slots, ntok, flat, opts, at, pool)
        assert_same(plain, snap)
        for s in snap[6]:
            s.free()


def launch_delta(m, slots, ntok, opts, at):
    V = m.info["num_vocab"]
    reset(m, slots)
    plain, snap = run_pair(m, slots, ntok, toks_for(sum(ntok), 31, V), opts, at)
    for s in snap[6]:
        s.free()
    return snap[5] - plain[5]


def test_launches_added_per_snapshot_step(models, ad_model):
    """The header's count: +1 row copy per step that holds a snapshot, +1 head launch when one of its snapshot tokens has no
    output row, +1 shrink in front of that launch on a step with a bound slot of an engine whose adapters touch the head."""
    m, _ = models("tiny6", max_batch=4, chunk=32)
    assert launch_delta(m, [0], [20], [FULL], [(0, 3), (0, 20)]) == 1
    assert launch_delta(m, [0], [20], [SCORE], [(0, 1), (0, 7)]) == 1
    assert launch_delta(m, [0], [20], [LAST], [(0, 20)]) == 1
    assert launch_delta(m, [0], [20], [NONE], [(0, 9)]) == 2
    assert launch_delta(m, [0], [20], [LAST], [(0, 4), (0, 20)]) == 2
    assert launch_delta(m, [0, 1], [10, 10], [FULL, NONE], [(0, 2), (1, 5)]) == 2
    # one entry of 100 tokens runs as steps of 32, 32, 32 and 4 tokens: the count scales with the steps holding snapshots
    assert launch_delta(m, [0], [100], [FULL], [(0, 1), (0, 40)]) == 2
    assert launch_delta(m, [0], [100], [FULL], [(0, 1), (0, 2), (0, 40), (0, 70), (0, 100)]) == 4
    assert launch_delta(m, [0], [100], [NONE], [(0, 10), (0, 40)]) == 4
    assert launch_delta(m, [0], [100], [NONE], [(0, 10), (0, 40), (0, 70), (0, 100)]) == 8
    assert launch_delta(m, [0], [100], [NONE], []) == 0
    assert launch_delta(m, [0], [100], [NONE], [(0, p) for p in range(1, 101)]) == 8
    ma = ad_model[0]
    assert launch_delta(ma, [0], [20], [NONE], [(0, 9)]) == 3        # slot 0 is bound
    assert launch_delta(ma, [0], [20], [FULL], [(0, 9)]) == 1
    assert launch_delta(ma, [1], [20], [NONE], [(0, 9)]) == 2        # slot 1 runs the base model


def test_reuse_list_must_match_the_snapshots(models):
    m, _ = models("tiny6", max_batch=2, chunk=32)
    with pytest.raises(ValueError):
        m.infer_snapshots([0], [4], [1, 2, 3, 4], [NONE], [(0, 1), (0, 2)], reuse=[None])


# ---- steps with more than 16 snapshot tokens without an output row (the snapshot head launch at 2, 4 and 8 token tiles) ----
def mtx_pair(m, n, orc=None, slot=0):
    """Call A: one NONE entry of n tokens with a snapshot at every token, in one step (chunk >= n); call B: the same tokens
    from the same state as FULL.  Both steps have T = n and mt_bucket(X) == mt_bucket(R), so A's snapshot head launch is B's
    head launch over other operand and output rows: every snapshot row equals B's logits row bit for bit, and every
    snapshot state B's snapshot at the same position.  A's other outputs equal infer_ex's; spot positions match the oracle."""
    V = m.info["num_vocab"]
    toks = toks_for(n, 500 + n, V)
    at = [(0, p) for p in range(1, n + 1)]
    reset(m, [slot])
    plain, snap_a = run_pair(m, [slot], [n], toks, [NONE], at)
    assert_same(plain, snap_a)
    reset(m, [slot])
    rows_b, _, snaps_b = m.infer_snapshots([slot], [n], toks, [FULL], at)
    for p, (sa, sb) in enumerate(zip(snap_a[6], snaps_b), 1):
        st_a, row_a = m.state.snapshot_back(sa, with_logits=True)
        st_b = m.state.snapshot_back(sb)
        assert np.array_equal(row_a, rows_b[0][p - 1]), f"position {p}: snapshot row != the FULL logits row"
        assert np.array_equal(st_a, st_b), f"position {p}: NONE and FULL snapshot states differ"
    if orc is not None:
        for p in sorted({1, 16, 17, n // 2, n}):
            check_snapshot(m, orc, snap_a[6][p - 1], toks, p)
    for s in list(snap_a[6]) + list(snaps_b):
        s.free()


@pytest.mark.parametrize("n", [17, 40, 100])
@pytest.mark.parametrize("preset", ["tiny6", "tiny7", "small6"])
def test_snapshot_head_over_token_tiles(models, preset, n):
    m, st = models(preset, max_batch=4, chunk=128)
    mtx_pair(m, n, O.Oracle(O.parse_st(st), "f16"))


def test_snapshot_head_over_token_tiles_bound_adapter():
    """The same on a bound slot of an engine whose adapter touches the head: the snapshot shrink runs over > 16 rows."""
    st = synth.make_st("tiny6", 0)
    ad = synth.make_lora_st("tiny6", rank=8, seed=11, targets=("att.key", "att.value", "ffn.key"))
    m = runtime.Model(st, max_batch=4, token_chunk_size=128, adapters=[(ad, 0.75)])
    try:
        m.bind_adapter([1], [1])
        w = O.parse_st(st)
        bound = AdapterOracle(w, "f16", (O.parse_st(ad), 0.75))
        for n in (17, 40, 100):
            mtx_pair(m, n, bound, slot=1)
    finally:
        m.close()


def test_snapshot_head_over_token_tiles_7b_layer_shape():
    """One layer at the 7B shape with the whole 65536-token vocabulary: the production head plan at 4 and 8 token tiles."""
    shp = dataclasses.replace(synth.PRESETS["v6-7b"], L=1)
    st = synth.make_st(shp, 0)
    m = runtime.Model(st, max_batch=1, token_chunk_size=128)
    try:
        assert m.info["num_vocab"] == 65536
        for n in (40, 100):
            mtx_pair(m, n)
    finally:
        m.close()
