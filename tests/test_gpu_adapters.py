"""Unblended LoRA adapters on the GPU (b200rwkv_create_adapters / b200rwkv_bind_adapter): the shrink kernel against a float64
reference (b200rwkv_op_adapter), bound slots against the oracle's unblended path, steps without a bound slot bit for bit
against a create_ex engine, and the readers of a bound slot's rows (SCORE, sample_topk, pooled hidden rows)."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

from adapter_oracle import AdapterOracle

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
ALPHA = (0.1, -0.15)
# two adapters of different ranks and targets (all eight projection kinds between them, and the head in both)
TARGETS = (("att.key", "att.value", "att.output", "ffn.key", "ffn.value"),
           ("att.receptance", "att.gate", "ffn.receptance", "ffn.value", "att.key"))


def rel_err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _f16_ulp(v):
    a = np.abs(v)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


# ---------------------------------------------------------------------------------------------------------------------------
# the shrink kernel
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("K", [256, 896, 1024, 512, 1792, 4096, 14336])
@pytest.mark.parametrize("T", [1, 16, 17, 128])
def test_shrink_kernel_matches_float64(T, K, precision):
    if precision == 1 and T > 16:
        pytest.skip("split operands are decode-shaped (<= 16 tokens)")
    rng = np.random.default_rng(T * 7919 + K + precision)
    ranks = [1, 8, 64, 128]
    mats = [(rng.standard_normal((K, r)) / np.sqrt(K)).astype(np.float16) for r in ranks]
    ids = rng.integers(0, len(ranks) + 1, size=T).astype(np.int32)
    ids[0] = 0
    if T > 1:
        ids[1] = 4
    x32 = (rng.standard_normal((T, K)) * 3).astype(np.float32)
    if precision == 0:
        x = x32.astype(np.float16)
        xv = x.astype(np.float64)
    else:
        hi = x32.astype(np.float16)
        lo = (x32 - hi.astype(np.float32)).astype(np.float16)
        x = np.stack([hi, lo], 0)
        xv = hi.astype(np.float64) + lo.astype(np.float64)
    tail = capi.op_adapter(x, mats, ids, precision=precision).astype(np.float64)
    got = tail if precision == 0 else tail[0] + tail[1]
    for t in range(T):
        for b in range(len(ranks)):
            if ids[t] != b + 1:
                assert not got[t, b].any(), (t, b)        # exact zeros in the other adapters' blocks
                if precision == 1:
                    assert not tail[1, t, b].any()
                continue
            r = ranks[b]
            A = mats[b].astype(np.float64)
            ref = xv[t] @ A
            acc = (K / 32 + 24) * 2.0 ** -24 * (np.abs(xv[t]) @ np.abs(A))     # f32 chains of K / 32 FMAs, 1 + 16 adds
            if precision == 0:
                bound = acc + _f16_ulp(ref) / 2 + 2.0 ** -25
            else:
                bound = acc + 2.0 ** -22 * np.abs(ref) + 2.0 ** -40
            err = np.abs(got[t, b, :r] - ref)
            assert (err <= bound).all(), (t, b, float((err / bound).max()))
            assert not got[t, b, r:].any()                # zeros above the rank


# ---------------------------------------------------------------------------------------------------------------------------
# engines
# ---------------------------------------------------------------------------------------------------------------------------
def _adapters(preset, ranks=(8, 16)):
    return [(synth.make_lora_st(preset, rank=r, seed=11 + i, targets=TARGETS[i]), ALPHA[i]) for i, r in enumerate(ranks)]


def _oracles(w, adapters, act="f16"):
    """oracle per adapter id: 0 = the base model"""
    return [O.Oracle(w, act)] + [AdapterOracle(w, act, adapter=(O.parse_st(img), a)) for img, a in adapters]


def _check(rows, want, state=None, want_state=None, tol=REL_TOL):
    assert rel_err(rows, want) <= tol
    assert np.array_equal(np.asarray(rows).argmax(-1), np.asarray(want).argmax(-1))
    if state is not None:
        assert rel_err(state, want_state) <= tol


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_bound_slots_match_the_oracle(preset):
    st = synth.make_st(preset, 0)
    w = O.parse_st(st)
    ads = _adapters(preset)
    orc = _oracles(w, ads)
    m = runtime.Model(st, max_batch=8, token_chunk_size=128, adapters=ads)
    rng = np.random.default_rng(3)
    V = m.info["num_vocab"]
    try:
        for s in range(8):
            m.state.load(m.state.init(), s)
        # decode-shaped steps for a slot bound to adapter 1
        m.bind_adapter([2], [1])
        toks = rng.integers(1, V, size=5).tolist()
        for t in toks:
            got = m.infer_raw([2], [1], [t], [capi.OPTION_LAST])[0]
        want, want_st = orc[1].run(toks, orc[1].state_init())
        _check(got, want, m.state.back(2), want_st)
        # one ragged call: slots on the base model, adapter 1 and adapter 2 (FULL rows)
        m.bind_adapter([0, 1, 3], [0, 1, 2])
        lens = {0: 3, 1: 7, 3: 5}
        seqs = {s: rng.integers(1, V, size=n).tolist() for s, n in lens.items()}
        for s in lens:
            m.state.load(m.state.init(), s)
        slots = [3, 0, 1]
        rows = m.infer_raw(slots, [lens[s] for s in slots], [t for s in slots for t in seqs[s]], [capi.OPTION_FULL] * 3)
        for i, (s, a) in enumerate(((3, 2), (0, 0), (1, 1))):
            want, want_st = orc[a].run(seqs[s], orc[a].state_init(), full=True)
            _check(rows[i], want, m.state.back(s), want_st)
        # prefill runs, bound to adapter 2, several of them in one call
        m.bind_adapter([4, 5, 6, 7], [2, 2, 1, 0])
        plens = [20, 50, 128, 300]
        pseq = [rng.integers(1, V, size=n).tolist() for n in plens]
        for s in (4, 5, 6, 7):
            m.state.load(m.state.init(), s)
        rows = m.infer_raw([4, 5, 6, 7], plens, [t for q in pseq for t in q], [capi.OPTION_LAST] * 4)
        for i, (s, a) in enumerate(((4, 2), (5, 2), (6, 1), (7, 0))):
            want, want_st = orc[a].run(pseq[i], orc[a].state_init())
            _check(rows[i], want, m.state.back(s), want_st)
        # rebinding mid-sequence: the slot continues from its state under the new adapter
        m.bind_adapter([2], [2])
        more = rng.integers(1, V, size=4).tolist()
        got = m.infer_raw([2], [4], more, [capi.OPTION_LAST])[0]
        _, mid = orc[1].run(toks, orc[1].state_init())
        want, want_st = orc[2].run(more, mid)
        _check(got, want, m.state.back(2), want_st)
        # state_load does not clear a binding
        m.state.load(m.state.init(), 2)
        got = m.infer_raw([2], [2], more[:2], [capi.OPTION_LAST])[0]
        want, _ = orc[2].run(more[:2], orc[2].state_init())
        _check(got, want)
    finally:
        m.close()


def test_precision1_bound_slots_match_the_f32_oracle():
    st = synth.make_st("tiny6", 0)
    w = O.parse_st(st)
    ads = _adapters("tiny6")
    orc = _oracles(w, ads, act="f32")
    m = runtime.Model(st, max_batch=4, token_chunk_size=32, precision=1, adapters=ads)
    rng = np.random.default_rng(9)
    try:
        seqs = [rng.integers(1, 512, size=n).tolist() for n in (1, 6, 20)]
        for s in range(3):
            m.state.load(m.state.init(), s)
        m.bind_adapter([0, 1, 2], [1, 2, 0])
        rows = m.infer_raw([0, 1, 2], [len(q) for q in seqs], [t for q in seqs for t in q], [capi.OPTION_LAST] * 3)
        for s, a in ((0, 1), (1, 2), (2, 0)):
            want, want_st = orc[a].run(seqs[s], orc[a].state_init())
            _check(rows[s], want, m.state.back(s), want_st)
    finally:
        m.close()


def _run_calls(m, rng_seed, V, S):
    """A fixed mix of calls: decode, ragged FULL / LAST / NONE, SCORE; returns every output and state."""
    rng = np.random.default_rng(rng_seed)
    out = []
    for s in range(S):
        m.state.load(m.state.init(), s)
    for _ in range(3):
        toks = rng.integers(1, V, size=S).tolist()
        out += m.infer_raw(list(range(S)), [1] * S, toks, [capi.OPTION_LAST] * S)
    lens = [5, 0, 40, 2]
    toks = rng.integers(1, V, size=sum(lens)).tolist()
    out += m.infer_raw([3, 1, 0, 2], lens, toks, [capi.OPTION_FULL, capi.OPTION_LAST, capi.OPTION_NONE, capi.OPTION_LAST])
    rows, scores = m.infer_ex([0, 1], [6, 3], rng.integers(1, V, size=9).tolist(), [capi.OPTION_SCORE, capi.OPTION_FULL])
    out += rows + [scores[0][0], scores[0][1].astype(np.float32)]
    out += [m.state.back(s) for s in range(S)]
    return out


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_unbound_steps_are_bit_identical_to_create_ex(preset):
    st = synth.make_st(preset, 0)
    ads = _adapters(preset)
    S = 4
    base_opts = runtime.Model(st, max_batch=S, token_chunk_size=64, devices=[0])
    ad = runtime.Model(st, max_batch=S, token_chunk_size=64, adapters=ads)
    V = ad.info["num_vocab"]
    try:
        n0 = base_opts.launch_count()
        want = _run_calls(base_opts, 4, V, S)
        d_want = base_opts.launch_count() - n0
        for rebind in (False, True):
            if rebind:           # bound, run, then bound to 0 again
                ad.bind_adapter([0, 2], [1, 2])
                _run_calls(ad, 5, V, S)
                ad.bind_adapter([0, 2], [0, 0])
            n1 = ad.launch_count()
            got = _run_calls(ad, 4, V, S)
            assert ad.launch_count() - n1 == d_want
            assert len(got) == len(want)
            for g, x in zip(got, want):
                assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(x).view(np.uint32))
    finally:
        for m in (base_opts, ad):
            m.close()


def test_a_bound_slot_composes_with_score_sampling_and_pooling():
    st = synth.make_st("small6", 0)
    ads = _adapters("small6")
    m = runtime.Model(st, max_batch=4, token_chunk_size=32, adapters=ads)
    rng = np.random.default_rng(21)
    V, C, L = m.info["num_vocab"], m.info["num_emb"], m.info["num_layer"]
    try:
        toks = rng.integers(1, V, size=37).tolist()
        for s in range(3):
            m.state.load(m.state.init(), s)
        m.bind_adapter([0, 1, 2], [1, 1, 2])
        # SCORE equals the log-softmax of the FULL rows of the same call (slot 0 FULL, slot 1 SCORE, same tokens and adapter)
        rows, scores = m.infer_ex([0, 1], [37, 37], toks + toks, [capi.OPTION_FULL, capi.OPTION_SCORE])
        full = rows[0].astype(np.float64)
        lsm = full - full.max(1, keepdims=True)
        lsm -= np.log(np.exp(lsm).sum(1, keepdims=True))
        want = lsm[np.arange(36), toks[1:]]
        assert np.abs(scores[1][0][1:] - want).max() <= 2e-5 * max(1.0, np.abs(want).max())
        assert np.array_equal(scores[1][1][1:], full[:-1].argmax(1))
        # sample_topk top-1 equals the argmax of the slot's kept row
        kept = m.infer_raw([2], [6], toks[:6], [capi.OPTION_LAST])[0][0]
        ids, _ = m.sample_topk([2], top_k=4)
        assert int(ids[0, 0]) == int(kept.argmax())
        # pooled hidden rows equal the per-token rows
        layer = L // 2
        for s in (0, 1):
            m.state.load(m.state.init(), s)
        m.keep_hidden(layers=[layer])
        m.keep_hidden_pooled([layer], mode="mean")
        m.infer_raw([0, 1], [20, 9], toks[:29], [capi.OPTION_NONE] * 2)
        per_tok = m.last_hidden(max_rows=29, layer=layer)
        pooled, _ = m.last_hidden_pooled(layer)
        ref = [per_tok[:20].astype(np.float32), per_tok[20:29].astype(np.float32)]
        for i, r in enumerate(ref):
            acc = np.zeros(C, np.float32)
            for row in r:
                acc = np.float32(acc + row)
            assert np.array_equal(pooled[i], (acc / np.float32(len(r))).astype(np.float32))
    finally:
        m.close()


def test_half_the_slots_bound_at_the_7b_layer_shape():
    """One layer with the 7B dimensions (C = 4096, F = 14336), batch 16, half the slots bound (two adapters at rank 64 and
    128), against the oracle."""
    shp = dataclasses.replace(synth.PRESETS["v6-7b"], L=1, V=4096)
    st = synth.make_st(shp, 0)
    w = O.parse_st(st)
    ads = _adapters(shp, ranks=(64, 128))
    orc = _oracles(w, ads)
    m = runtime.Model(st, max_batch=16, token_chunk_size=64, adapters=ads)
    try:
        rng = np.random.default_rng(5)
        toks = rng.integers(1, 4000, size=(16, 3))
        slots = list(range(16))
        bind = [1 if s % 4 == 0 else (2 if s % 4 == 1 else 0) for s in slots]
        m.bind_adapter(slots, bind)
        for s in slots:
            m.state.load(m.state.init(), s)
        for j in range(3):
            rows = m.infer_raw(slots, [1] * 16, toks[:, j].tolist(), [capi.OPTION_LAST] * 16)
        for s in (0, 1, 2, 5, 15):
            a = bind[s]
            want, want_st = orc[a].run(toks[s].tolist(), orc[a].state_init())
            _check(rows[s][0], want[0], m.state.back(s), want_st)
        ptoks = rng.integers(1, 4000, size=40).tolist()
        m.state.load(m.state.init(), 1)
        got = m.infer_raw([1], [40], ptoks, [capi.OPTION_LAST])[0][0]
        want, _ = orc[2].run(ptoks, orc[2].state_init())
        _check(got, want[0])
    finally:
        m.close()


def test_engine_refusals():
    st = synth.make_st("tiny6", 0)
    ads = _adapters("tiny6")
    m = runtime.Model(st, max_batch=4, token_chunk_size=32, adapters=ads)
    try:
        for slots, ids, code in (([4], [1], capi.ERR_STATE), ([0], [3], capi.ERR_INVALID), ([0, 1, 2, 3, 0], [0] * 5, capi.ERR_INVALID),
                                 ([0, 0], [1, 2], capi.ERR_INVALID)):
            with pytest.raises(capi.B200Error) as ei:
                m.bind_adapter(slots, ids)
            assert ei.value.code == code, (slots, ids)
    finally:
        m.close()
    # a pair on a matrix of a quantised layer
    with pytest.raises(capi.B200Error) as ei:
        runtime.Model(st, max_batch=2, quant=1, quant_type="Int8", adapters=ads)
    assert ei.value.code == capi.ERR_UNSUPPORTED


def test_two_devices_are_refused():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    st = synth.make_st("tiny6", 0)
    with pytest.raises(capi.B200Error) as ei:
        runtime.Model(st, max_batch=2, devices=[0, 1], adapters=_adapters("tiny6"))
    assert ei.value.code == capi.ERR_UNSUPPORTED
