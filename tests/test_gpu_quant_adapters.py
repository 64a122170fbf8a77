"""GPU tests of adapters on quantised layers (b200rwkv_options.quant_adapters) for Int8, NF4, FP8 and Int4: one W' launch
through b200rwkv_op_gemm_tail against float64 (codes times the format's dequantised weights, FP8 rows scaled, plus the f16
tail terms unscaled) over token tiles, tail counts, every activation and both output modes, and forced stream-K grids whose
cuts fall on the code / tail boundary, inside the tail and across it; engines with every layer quantised against
AdapterOracle on the dequantised weights; the bits of unbound steps against create_ex; places against create_adapters; and a
bound slot through SCORE, sample_topk, pooled hidden rows and snapshots."""
import dataclasses
import zlib

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q
from oracle import rwkv_numpy as O

import fp8_oracle as F
import int4_oracle as I
import test_gpu_gemm as G
from adapter_oracle import AdapterOracle
from test_gpu_adapters import ALPHA, TARGETS
from test_gpu_quant import rel_err

pytestmark = pytest.mark.gpu

QUANTS = [capi.QUANT_INT8, capi.QUANT_NF4, capi.QUANT_FP8, capi.QUANT_INT4]
REL_TOL = 1e-3


def _dequant(w, qt):
    if qt == capi.QUANT_NONE:
        return w.astype(np.float64)
    if qt == capi.QUANT_INT8:
        return Q.dequant_int8(*Q.quant_int8(w), contract="engine").astype(np.float64)
    if qt == capi.QUANT_NF4:
        return Q.dequant_nf4(*Q.quant_nf4(w), contract="engine").astype(np.float64)
    if qt == capi.QUANT_FP8:
        return F.dequant_fp8(*F.quant_fp8(w)).astype(np.float64)
    return I.dequant_int4(*I.quant_int4(w)).astype(np.float64)


def _quantize_model(w, layers, qt):
    return I.quantize_model(w, layers, qt) if qt == capi.QUANT_INT4 else F.quantize_model(w, layers, qt)


# ----------------------------------------------------------------------------------------------------------------------
# one W' launch against float64
# ----------------------------------------------------------------------------------------------------------------------
def _run_tail(qt, T, n, N=256, K=512, act=capi.ACT_NONE, mode=capi.OUT_F32, grid=0, bias=True):
    rng = np.random.default_rng(zlib.crc32(repr((qt, T, n, N, K, act, mode, grid)).encode()))
    w = G.weights(N, K, 7, edge=True)
    x = rng.standard_normal((1, T, K), dtype=np.float32)
    e = (rng.standard_normal((N, 128 * n), dtype=np.float32) * np.float32(0.05)).astype(np.float16)
    u = rng.standard_normal((T, 128 * n), dtype=np.float32).astype(np.float16)
    rows = capi.gemm_rows(T)
    a16 = mode != capi.OUT_F32
    out = np.empty((1, rows, N + 8), np.uint16 if a16 else np.float32)
    out.view(np.uint16 if a16 else np.uint32)[...] = G.SENT16 if a16 else G.SENT32
    b = rng.standard_normal(N, dtype=np.float32) * np.float32(0.5) if bias else None
    plan = capi.op_gemm_tail(T, dict(w=w, x=x, bias=b, act=act, out_mode=mode, out=out), e, u, quant_type=qt, grid=grid)
    # the float64 reference over the extended operand [x | u] and matrix [W^ | e]: the codes' part with the format's
    # dequantised weights (s_n value(q) for FP8), the tail part unscaled, in the projection tests' bound
    wx = np.concatenate([_dequant(w, qt), e.astype(np.float64)], axis=1)
    xx = np.concatenate([x[0].astype(np.float16).astype(np.float64), u.astype(np.float64)], axis=1)
    y, bound = G.project64(xx, wx, b, act)
    written = np.zeros(out.shape[1:], bool)
    written[:T, :N] = True
    if a16:
        got = out[0, :T, :N].view(np.float16).astype(np.float64)
        y = np.clip(y, -G.F16_MAX, G.F16_MAX)
        bound = bound + np.minimum(np.spacing(np.abs(y).astype(np.float16)).astype(np.float64), 32.0)
        sent = out.view(np.uint16)[0][~written] == G.SENT16
    else:
        got = out[0, :T, :N].astype(np.float64)
        sent = out.view(np.uint32)[0][~written] == G.SENT32
    ratio = np.abs(got - y) / bound
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    assert ratio.max() <= 1.0, (qt, T, n, grid, float(ratio.max()))
    assert sent.all(), "a cell outside [T, N] was written"
    if act == capi.ACT_NONE:               # the tail is really there: without it most outputs are off by far more than the bound
        y0, _ = G.project64(xx[:, :K], wx[:, :K], b, act)
        assert (np.abs(y0 - y) > 10 * bound).mean() > 0.5
    return plan


@pytest.mark.parametrize("n", [1, 8])
@pytest.mark.parametrize("T", [1, 16, 17, 64, 128])
@pytest.mark.parametrize("qt", [capi.QUANT_NONE] + QUANTS)
def test_tail_launch_token_tiles(qt, T, n):
    _run_tail(qt, T, n)


@pytest.mark.parametrize("mode", [capi.OUT_F32, capi.OUT_A16])
@pytest.mark.parametrize("act", range(capi.ACT_V7DECAY + 1))
@pytest.mark.parametrize("qt", QUANTS)
def test_tail_launch_every_activation_and_output_mode(qt, act, mode):
    _run_tail(qt, 17, 1, act=act, mode=mode)


# N = 256, K = 512: two tiles of 4 code blocks and n tail blocks each
#   n = 1, grid 5: cuts at 2, 4, 6, 8 -- CTA 2 holds tile 0's tail block alone (a tail-only contributor), cut 4 is exactly
#     tile 0's code / tail boundary;
#   n = 8, grid 3: cuts at 8 (inside tile 0's tail) and 16 (tile 1's code / tail boundary);
#   n = 8, grid 7 and one block per CTA: cuts across every boundary, most contributors of a tile tail-only.
@pytest.mark.parametrize("n,grid", [(1, 5), (1, 3), (1, 10), (8, 3), (8, 7), (8, 24)])
@pytest.mark.parametrize("T", [1, 16, 64])
@pytest.mark.parametrize("qt", QUANTS)
def test_tail_launch_stream_k_cuts(qt, T, n, grid):
    plan = _run_tail(qt, T, n, grid=grid)
    assert plan[:3] == (grid, 2 * (4 + n), 2)


# ----------------------------------------------------------------------------------------------------------------------
# engines
# ----------------------------------------------------------------------------------------------------------------------
def _check(got, want, st, want_st):
    assert rel_err(got, want) <= REL_TOL
    assert (np.atleast_2d(got).argmax(-1) == np.atleast_2d(want).argmax(-1)).all()
    assert rel_err(st, want_st) <= REL_TOL


@pytest.mark.parametrize("preset", ["tiny6", "tiny5", "tiny7", "small6"])
@pytest.mark.parametrize("qt", QUANTS)
def test_create_adapters_engines_match_the_oracle(qt, preset):
    """Every layer quantised; slots bound to adapter 1, adapter 2 and none in one call."""
    shape = synth.PRESETS[preset]
    st = synth.make_st(shape, 0)
    w = O.parse_st(st)
    wq = _quantize_model(w, shape.L, qt)
    # test_gpu_adapters' pair: all eight projection kinds between them, the head in both
    ads = [(synth.make_lora_st(shape, rank=r, seed=11 + i, targets=TARGETS[i]), ALPHA[i]) for i, r in enumerate((8, 32))]
    m = runtime.Model(st, max_batch=4, token_chunk_size=64, quant=shape.L, quant_type=qt, adapters=ads, quant_adapters=True)
    try:
        orcs = [O.Oracle(wq, "f16")] + [AdapterOracle(wq, "f16", adapter=(O.parse_st(img), a)) for img, a in ads]
        for s in range(3):
            m.state.load(m.state.init(), s)
        m.bind_adapter([0, 1, 2], [1, 2, 0])
        seqs = {0: [1, 5, 9, 33, 2], 1: [7, 300, 41], 2: [41, 8, 0, 17]}
        rows = m.infer_raw([0, 1, 2], [len(seqs[s]) for s in range(3)], [t for s in range(3) for t in seqs[s]],
                           [capi.OPTION_FULL] * 3)
        for s, a in ((0, 1), (1, 2), (2, 0)):
            want, want_st = orcs[a].run(seqs[s], orcs[a].state_init(), full=True)
            _check(rows[s], want, m.state.back(s), want_st)
        # the adapter is really in effect on the quantised layers
        plain, _ = orcs[0].run(seqs[0], orcs[0].state_init(), full=True)
        assert rel_err(rows[0], plain) > 2 * REL_TOL
    finally:
        m.close()


@pytest.mark.parametrize("qt", QUANTS)
def test_places_with_some_layers_quantised(qt):
    """quant_layers = 1: a place reaches the quantised layer 0, the f16 layers and the head; a place loaded with file F at
    id i gives the bits of create_adapters with F at i."""
    shape = synth.PRESETS["tiny6"]
    st = synth.make_st(shape, 0)
    w = O.parse_st(st)
    # the places engine targets exactly the kinds the files pair, so both engines hold the same plans
    f = synth.make_lora_st(shape, rank=16, seed=3, targets=TARGETS[1])
    kw = dict(max_batch=2, token_chunk_size=64, quant=1, quant_type=qt, quant_adapters=True)
    mp = runtime.Model(st, adapter_places=2, adapter_targets=TARGETS[1] + ("head",), **kw)
    ma = runtime.Model(st, adapters=[(synth.make_lora_st(shape, rank=4, seed=9, targets=TARGETS[1]), 0.1), (f, 0.15)], **kw)
    try:
        mp.load_adapter(2, f, 0.15)
        toks = [3, 1, 4, 1, 5, 9, 2, 6]
        outs = []
        for m in (mp, ma):
            m.state.load(m.state.init(), 0)
            m.bind_adapter([0], [2])
            outs.append((m.infer_raw([0], [len(toks)], toks, [capi.OPTION_FULL])[0].copy(), m.state.back(0)))
        assert np.array_equal(outs[0][0].view(np.uint32), outs[1][0].view(np.uint32))
        assert np.array_equal(outs[0][1].view(np.uint32), outs[1][1].view(np.uint32))
        orc = AdapterOracle(_quantize_model(w, 1, qt), "f16", adapter=(O.parse_st(f), 0.15))
        want, want_st = orc.run(toks, orc.state_init(), full=True)
        _check(outs[0][0], want, outs[0][1], want_st)
        # unload: the place's slot is the base model again
        mp.bind_adapter([0], [0])
        mp.unload_adapter(2)
        mp.state.load(mp.state.init(), 0)
        got = mp.infer_raw([0], [len(toks)], toks, [capi.OPTION_FULL])[0]
        base, _ = O.Oracle(_quantize_model(w, 1, qt), "f16").run(toks, orc.state_init(), full=True)
        assert rel_err(got, base) <= REL_TOL
    finally:
        mp.close()
        ma.close()


def _unbound_run(m, bind):
    """Two slots, a prompt and three decode steps with SCORE; returns logits, states and scores as bits, and launches."""
    toks = [[5, 6, 7, 8, 9, 10], [11, 12, 13]]
    for s in range(2):
        m.state.load(m.state.init(), s)
    if bind:
        m.bind_adapter([0, 1], [1, 0])
        m.bind_adapter([0], [0])
    n0 = m.launch_count()
    rows = m.infer_raw([0, 1], [6, 3], toks[0] + toks[1], [capi.OPTION_FULL, capi.OPTION_LAST])
    res = [r.copy().view(np.uint32) for r in rows]
    for t in (20, 21, 22):
        res += [r.copy().view(np.uint32) for r in m.infer_raw([0, 1], [1, 1], [t, t + 1], [capi.OPTION_LAST] * 2)]
    _, scores = m.infer_ex([0, 1], [3, 2], [1, 2, 3, 4, 5], [capi.OPTION_SCORE] * 2)
    res += [np.asarray(v).copy().view(np.uint32) for sc in scores for v in sc]
    res += [m.state.back(s).view(np.uint32) for s in range(2)]
    return res, m.launch_count() - n0


@pytest.mark.parametrize("qt", QUANTS)
def test_unbound_steps_are_create_ex_bit_for_bit(qt):
    shape = synth.PRESETS["tiny6"]
    st = synth.make_st(shape, 0)
    kw = dict(max_batch=2, token_chunk_size=64, quant=shape.L, quant_type=qt)
    base = runtime.Model(st, **kw)
    ad = runtime.Model(st, adapters=[(synth.make_lora_st(shape, rank=8, seed=1), 1.0)], quant_adapters=True, **kw)
    try:
        want, n_want = _unbound_run(base, False)
        for bind in (False, True):          # before any binding, and after a bind and an unbind
            got, n_got = _unbound_run(ad, bind)
            assert n_got == n_want
            assert len(got) == len(want)
            for a, b in zip(got, want):
                assert np.array_equal(np.asarray(a), np.asarray(b))
    finally:
        base.close()
        ad.close()


def test_flag_without_quantised_layers_changes_nothing():
    shape = synth.PRESETS["tiny6"]
    st = synth.make_st(shape, 0)
    ads = [(synth.make_lora_st(shape, rank=8, seed=1), 1.0)]
    ms = [runtime.Model(st, max_batch=2, token_chunk_size=64, adapters=ads, quant_adapters=q) for q in (False, True)]
    try:
        outs = []
        for m in ms:
            m.state.load(m.state.init(), 0)
            m.bind_adapter([0], [1])
            n0 = m.launch_count()
            r = m.infer_raw([0], [5], [1, 2, 3, 4, 5], [capi.OPTION_FULL])[0].copy()
            outs.append((r.view(np.uint32), m.state.back(0).view(np.uint32), m.launch_count() - n0))
        assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
        assert outs[0][2] == outs[1][2]
    finally:
        for m in ms:
            m.close()


@pytest.mark.parametrize("qt", [capi.QUANT_FP8, capi.QUANT_INT4])
def test_bound_slot_composes_with_score_sampling_pooling_and_snapshots(qt):
    shape = synth.PRESETS["tiny6"]
    st = synth.make_st(shape, 0)
    w = O.parse_st(st)
    f = synth.make_lora_st(shape, rank=8, seed=5)
    m = runtime.Model(st, max_batch=2, token_chunk_size=64, quant=shape.L, quant_type=qt, adapters=[(f, 0.1)],
                      quant_adapters=True)
    try:
        orc = AdapterOracle(_quantize_model(w, shape.L, qt), "f16", adapter=(O.parse_st(f), 0.1))
        toks = [4, 8, 15, 16, 23, 42]
        m.bind_adapter([0], [1])
        # SCORE: the scores of tokens 1.. given their prefixes, against the oracle's log-softmax
        m.state.load(m.state.init(), 0)
        full = m.infer_raw([0], [len(toks)], toks, [capi.OPTION_FULL])[0].copy()
        want, _ = orc.run(toks, orc.state_init(), full=True)
        assert rel_err(full, want) <= REL_TOL
        m.state.load(m.state.init(), 0)
        m.infer_raw([0], [1], toks[:1], [capi.OPTION_LAST])
        _, scores = m.infer_ex([0], [len(toks) - 1], toks[1:], [capi.OPTION_SCORE])
        score, argmax = scores[0]
        score = np.asarray(score, np.float64)
        lsm = want[:-1] - np.log(np.exp(want[:-1] - want[:-1].max(1, keepdims=True)).sum(1, keepdims=True)) - want[:-1].max(1, keepdims=True)
        ref = lsm[np.arange(len(toks) - 1), toks[1:]]
        assert np.abs(score - ref).max() <= 1e-2
        assert (np.asarray(argmax) == want[:-1].argmax(1)).all()
        # sample_topk over the kept row of the bound slot: the best candidate is the oracle's argmax
        m.state.load(m.state.init(), 0)
        m.infer_raw([0], [len(toks)], toks, [capi.OPTION_LAST])
        ids, _ = m.sample_topk([0], top_k=4)
        assert int(np.asarray(ids).reshape(-1)[0]) == int(want[-1].argmax())
        # pooled hidden rows: the bound slot's last-token row equals the recorded hidden row of a plain call
        m.keep_hidden_pooled([shape.L - 1], mode="last")
        m.state.load(m.state.init(), 0)
        m.infer_raw([0], [len(toks)], toks, [capi.OPTION_LAST])
        pooled = m.last_hidden_pooled(shape.L - 1)[0][0].copy()
        m.keep_hidden_pooled([])
        m.state.load(m.state.init(), 0)
        m.infer_raw([0], [len(toks)], toks, [capi.OPTION_LAST])
        last = m.last_hidden(64)[-1]
        assert np.array_equal(np.asarray(pooled).reshape(-1).view(np.uint32), np.asarray(last).reshape(-1).view(np.uint32))
        # snapshots: the snapshot at token 3 equals state_read at that boundary
        m.state.load(m.state.init(), 0)
        _, _, snaps = m.infer_snapshots([0], [len(toks)], toks, [capi.OPTION_LAST], [(0, 3)])
        snap, row = m.state.snapshot_back(snaps[0], with_logits=True)
        m.state.load(m.state.init(), 0)
        r3 = m.infer_raw([0], [3], toks[:3], [capi.OPTION_LAST])[0].copy()
        assert np.array_equal(np.asarray(snap).view(np.uint32), m.state.back(0).view(np.uint32))
        assert np.array_equal(np.asarray(row).reshape(-1).view(np.uint32), r3.reshape(-1).view(np.uint32))
    finally:
        m.close()


def test_7b_layer_at_batch_16_half_bound():
    """The 7B layer shape (C 4096, F 14336), one Int4 layer with adapters on every kind, 16 slots, half bound."""
    shape = dataclasses.replace(synth.PRESETS["v6-7b"], L=1, V=4096)
    st = synth.make_st(shape, 0)
    w = O.parse_st(st)
    f = synth.make_lora_st(shape, rank=64, seed=1)
    m = runtime.Model(st, max_batch=16, token_chunk_size=64, quant=1, quant_type="Int4", adapters=[(f, 1.0)],
                      quant_adapters=True)
    try:
        wq = _quantize_model(w, 1, capi.QUANT_INT4)
        orcs = [O.Oracle(wq, "f16"), AdapterOracle(wq, "f16", adapter=(O.parse_st(f), 1.0))]
        slots = list(range(16))
        for s in slots:
            m.state.load(m.state.init(), s)
        m.bind_adapter(slots, [s % 2 for s in slots])
        toks = np.random.default_rng(7).integers(1, 4000, size=(16, 3))
        for j in range(3):
            rows = m.infer_raw(slots, [1] * 16, toks[:, j].tolist(), [capi.OPTION_LAST] * 16)
        for s in (0, 1, 14, 15):
            o = orcs[s % 2]
            want, want_st = o.run(toks[s].tolist(), o.state_init())
            _check(rows[s][0], want, m.state.back(s), want_st)
    finally:
        m.close()
