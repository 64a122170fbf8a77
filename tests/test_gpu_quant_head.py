"""GPU tests of the quantised vocabulary head (b200rwkv_head_format): the projection kernels at the head's shapes against
float64 on the dequantised matrix (tests/test_gpu_gemm.py's bound); engines with a quantised head, with f16 and with Int4
layers, against the forward-pass oracle on tests/head_oracle.quantize_head(quantize_model(...)) (1e-3 relative, argmax equal
but for near-ties); NONE giving back the f16 head's bits; snapshot rows, SCORE and score_top reading the rows the quantised head wrote; batch-invariant
engines; weight updates against fresh engines; adapters; refusals; and the step's weight bytes."""
import functools

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

from adapter_oracle import AdapterOracle
import fp8_oracle as F8
import head_oracle as H
import int4_oracle as I4
import test_gpu_gemm as G
from test_gpu_quant import feed, rel_err
from test_gpu_score import check_scores, primed_snapshot

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
FORMATS = {"Int8": capi.QUANT_INT8, "NF4": capi.QUANT_NF4, "FP8": capi.QUANT_FP8, "Int4": capi.QUANT_INT4}


def oracle(w, head, layers=0, layer_type=capi.QUANT_NONE):
    wq = H.QUANTIZE[layer_type](w, layers, layer_type) if layers else w
    return O.Oracle(H.quantize_head(wq, head), "f16")


def argmax_agrees(got, want):
    """Argmax equal on every row, except where the oracle's row holds a near-tie: the engine's pick is within the 1e-3
    tolerance of the oracle's maximum (the two sum in different orders).  Such rows must stay rare."""
    g, w = got.argmax(1), want.argmax(1)
    rows = np.nonzero(g != w)[0]
    tol = 2 * REL_TOL * np.abs(want).max()
    ties = all(want[r, w[r]] - want[r, g[r]] <= tol for r in rows)
    return ties and len(rows) <= max(1, len(g) // 20)


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


# ----------------------------------------------------------------------------------------------------------------------
# the projection kernels at the head's shapes
# ----------------------------------------------------------------------------------------------------------------------
_dequantised_int = G.dequantised


@functools.lru_cache(maxsize=2)
def _dequantised(N, K, seed, edge, qtype):
    w = G.weights(N, K, seed, edge)
    if qtype == capi.QUANT_FP8:
        return F8.dequant_fp8(*F8.quant_fp8(w))
    if qtype == capi.QUANT_INT4:
        return I4.dequant_int4(*I4.quant_int4(w))
    return _dequantised_int(N, K, seed, edge, qtype)


@pytest.fixture(autouse=True)
def _format_reference_weights(monkeypatch):
    """test_gpu_gemm's float64 reference multiplies with each format's dequantised weights."""
    monkeypatch.setattr(G, "dequantised", _dequantised)


@pytest.mark.parametrize("T", [1, 16, 128])
@pytest.mark.parametrize("K", [4096, 2560])
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_head_shape_launches(fmt, K, T):
    """N = 65536: the vocabulary head of the 7B / 3B (K 4096, 2560) and RWKV-7 2.9B (K 2560) models, on the engine's plan."""
    plan = G.run("qhead", T, [G.seg(65536, K, pad=0)], quant=FORMATS[fmt], launches=1)
    assert plan[1:3] == (512 * K // 128, 512)


# ----------------------------------------------------------------------------------------------------------------------
# engines with a quantised head
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def image():
    cache = {}

    def get(preset, seed=0):
        if (preset, seed) not in cache:
            st = synth.make_st(synth.PRESETS[preset], seed)
            cache[(preset, seed)] = (st, O.parse_st(st))
        return cache[(preset, seed)]
    return get


@pytest.mark.parametrize("layers", ["f16", "Int4"])
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_logits_match_the_oracle(image, preset, fmt, layers):
    st, w = image(preset)
    L = synth.PRESETS[preset].L if layers == "Int4" else 0
    m = runtime.Model(st, max_batch=4, token_chunk_size=64, quant=L, quant_type=layers if L else 0, quant_head=fmt)
    try:
        orc = oracle(w, FORMATS[fmt], L, capi.QUANT_INT4 if L else capi.QUANT_NONE)
        toks = [1, 5, 9, 33, 2, 7, 300, 41, 41, 8, 0, 17]
        m.state.load(m.state.init(), 0)
        got = np.stack([feed(m, 0, [t])[0] for t in toks])              # decode steps
        want, want_state = orc.run(toks, orc.state_init(), full=True)
        assert rel_err(got, want) <= REL_TOL
        assert argmax_agrees(got, want)
        assert rel_err(m.state.back(0), want_state) <= REL_TOL
        # a ragged prefill: FULL rows of three entries of different lengths in one call
        rng = np.random.default_rng(4)
        seqs = [rng.integers(1, 500, n).tolist() for n in (70, 3, 21)]
        for s in range(3):
            m.state.load(m.state.init(), s)
        rows = m.infer_raw([0, 1, 2], [len(x) for x in seqs], [t for x in seqs for t in x], [capi.OPTION_FULL] * 3)
        for s, x in enumerate(seqs):
            want, _ = orc.run(x, orc.state_init(), full=True)
            assert rel_err(rows[s], want) <= REL_TOL, s
            assert argmax_agrees(rows[s], want), s
        # the format is really in effect: the f16 head answers differently
        plain, _ = oracle(w, capi.QUANT_NONE, L, capi.QUANT_INT4 if L else capi.QUANT_NONE).run(toks, orc.state_init(), full=True)
        want, _ = orc.run(toks, orc.state_init(), full=True)
        assert rel_err(want, plain) > 1e-4
    finally:
        m.close()


def _work(m):
    """Rows, states and per-step launch counts of a fixed mix of decode and prefill steps from the initial state."""
    rng = np.random.default_rng(9)
    out, counts = [], []
    for s in range(3):
        m.state.load(m.state.init(), s)
    for ntok, opt in (([1, 1, 1], capi.OPTION_LAST), ([40, 7, 1], capi.OPTION_FULL), ([1, 1, 1], capi.OPTION_LAST)):
        toks = rng.integers(1, 500, sum(ntok)).tolist()
        n0 = m.launch_count()
        rows = m.infer_raw([0, 1, 2], ntok, toks, [opt] * 3)
        counts.append(m.launch_count() - n0)
        out += [r.copy() for r in rows]
    return out, [m.state.back(s) for s in range(3)], counts


def test_none_gives_back_the_f16_head(image):
    st, _ = image("tiny6")
    ref = runtime.Model(st, max_batch=4, token_chunk_size=64)
    m = runtime.Model(st, max_batch=4, token_chunk_size=64)
    try:
        rows0, states0, counts0 = _work(ref)
        m.head_format("FP8")
        rows_q, _, counts_q = _work(m)
        assert counts_q == counts0                          # a quantised head launches as many kernels as the f16 head
        assert not all(same_bits(a, b) for a, b in zip(rows_q, rows0))
        m.head_format("FP8")                                # the current format again: nothing changes
        rows_q2, _, _ = _work(m)
        assert all(same_bits(a, b) for a, b in zip(rows_q, rows_q2))
        m.head_format("None")
        rows1, states1, counts1 = _work(m)
        assert all(same_bits(a, b) for a, b in zip(rows1, rows0))
        assert all(same_bits(a, b) for a, b in zip(states1, states0))
        assert counts1 == counts0
    finally:
        m.close()
        ref.close()


def test_switching_formats_matches_engines_created_with_them(image):
    st, _ = image("tiny7")
    m = runtime.Model(st, max_batch=4, token_chunk_size=64)
    try:
        for fmt in ("Int8", "Int4", "NF4", "FP8"):
            m.head_format(fmt)
            got, states, _ = _work(m)
            fresh = runtime.Model(st, max_batch=4, token_chunk_size=64, quant_head=fmt)
            try:
                want, want_states, _ = _work(fresh)
            finally:
                fresh.close()
            assert all(same_bits(a, b) for a, b in zip(got, want)), fmt
            assert all(same_bits(a, b) for a, b in zip(states, want_states)), fmt
    finally:
        m.close()


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_snapshot_rows_scores_and_score_top(image, preset):
    st, _ = image(preset)
    m = runtime.Model(st, max_batch=4, token_chunk_size=64, quant_head="Int4")
    try:
        rng = np.random.default_rng(3)
        toks = rng.integers(1, 500, 40).tolist()
        m.state.load(m.state.init(), 0)
        full = m.infer_raw([0], [40], toks, [capi.OPTION_FULL])[0].copy()
        # snapshot rows: the head launch of the snapshot tokens gives the bits of the same tokens' FULL rows
        at = [3, 17, 29, 40]
        m.state.load(m.state.init(), 1)
        _, _, snaps = m.infer_snapshots([1], [40], toks, [capi.OPTION_LAST], [(0, p) for p in at])
        for p, sn in zip(at, snaps):
            _, row = m.state.snapshot_back(sn, with_logits=True)
            assert same_bits(row, full[p - 1]), p
            sn.free()
        # SCORE values and score_top lists from the rows the quantised head wrote
        snap = primed_snapshot(m, 2, rng)
        _, kept0 = m.state.snapshot_back(snap, with_logits=True)
        m.state.write(snap, 2)
        rows = m.infer_raw([2], [len(toks)], toks, [capi.OPTION_FULL])[0].copy()
        m.state.write(snap, 2)
        _, sc, tops = m.infer_ex([2], [len(toks)], toks, [capi.OPTION_SCORE], top_n=5)
        scores, argmax = sc[0]
        check_scores(f"qhead/{preset}", scores, argmax, [kept0] + list(rows[:-1]), toks)
        ids, lps = tops[0]
        for j, row in enumerate([kept0] + list(rows[:-1])):
            order = np.lexsort((np.arange(row.size), -row.astype(np.float64)))[:5]
            assert ids[j].tolist() == order.tolist(), j
            if toks[j] in ids[j].tolist():
                assert same_bits(lps[j][ids[j].tolist().index(toks[j])], scores[j])
        snap.free()
    finally:
        m.close()


@pytest.mark.parametrize("fmt", ["FP8", "Int4"])
def test_batch_invariant_engine(image, fmt):
    """A 300-token FULL prompt (steps of 128, 128 and 44 tokens) gives the bits of the same tokens fed one per call."""
    st, _ = image("tiny6")
    m = runtime.Model(st, max_batch=4, token_chunk_size=128, batch_invariant=True, quant_head=fmt)
    try:
        for s in range(2):
            m.state.load(m.state.init(), s)
        toks = np.random.default_rng(1).integers(1, m.info["num_vocab"], size=300).tolist()
        full = m.infer_raw([0], [300], toks, [capi.OPTION_FULL])[0].copy()
        ref = np.stack([m.infer_raw([1], [1], [t], [capi.OPTION_LAST])[0][0].copy() for t in toks])
        assert same_bits(full, ref)
        assert same_bits(m.state.back(0), m.state.back(1))
    finally:
        m.close()


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_weight_updates_equal_creation(image, fmt):
    st0, _ = image("tiny6", 0)
    st1, w1 = image("tiny6", 1)
    m = runtime.Model(st0, max_batch=4, token_chunk_size=64, quant_head=fmt)
    fresh = runtime.Model(st1, max_batch=4, token_chunk_size=64, quant_head=fmt)
    try:
        m.update_weights(st1)
        got, states, counts = _work(m)
        want, want_states, want_counts = _work(fresh)
        assert all(same_bits(a, b) for a, b in zip(got, want))
        assert all(same_bits(a, b) for a, b in zip(states, want_states)) and counts == want_counts
        # head.weight alone, from the device: the codes follow it
        import torch
        m.update_weights(st0)
        m.update_weights_from_tensors({"head.weight": torch.from_numpy(w1["head.weight"].copy()).cuda()})
        merged = synth.pack_st({**O.parse_st(st0), "head.weight": w1["head.weight"]})
        fresh2 = runtime.Model(merged, max_batch=4, token_chunk_size=64, quant_head=fmt)
        try:
            got, _, _ = _work(m)
            want, _, _ = _work(fresh2)
            assert all(same_bits(a, b) for a, b in zip(got, want))
        finally:
            fresh2.close()
    finally:
        m.close()
        fresh.close()


@pytest.mark.parametrize("how", ["file", "place"])
def test_adapters_without_a_head_pair_use_the_quantised_head(image, how):
    """Bound and unbound slots, on an engine from create_adapters whose file pairs no head, and on a places engine that does
    not target the head, against the unblended adapter oracle with the Int8 head."""
    st, w = image("tiny6")
    lora = O.parse_st(synth.make_lora_st("tiny6", rank=8, seed=1))
    lora = {k: v for k, v in lora.items() if not k.startswith("head.")}
    img = synth.pack_st(lora)
    if how == "file":
        m = runtime.Model(st, max_batch=4, token_chunk_size=64, adapters=[(img, 1.0)], quant_head="Int8")
    else:
        m = runtime.Model(st, max_batch=4, token_chunk_size=64, adapter_places=1, adapter_targets=("att.key", "ffn.value"),
                          quant_head="Int8")
        lora = {k: v for k, v in lora.items() if ".att.key." in k or ".ffn.value." in k}
        m.load_adapter(1, synth.pack_st(lora), 1.0)
    try:
        m.bind_adapter([0], [1])
        wq = H.quantize_head(w, capi.QUANT_INT8)
        toks = [1, 5, 9, 33, 2, 7]
        for s in range(2):
            m.state.load(m.state.init(), s)
        rows = m.infer_raw([0, 1], [6, 6], toks + toks, [capi.OPTION_FULL] * 2)
        for s, orc in enumerate((AdapterOracle(wq, "f16", (lora, 1.0)), AdapterOracle(wq, "f16"))):
            want, _ = orc.run(toks, orc.state_init(), full=True)
            assert rel_err(rows[s], want) <= REL_TOL and argmax_agrees(rows[s], want), s
    finally:
        m.close()


@pytest.mark.parametrize("how", ["pair", "place"])
def test_engines_whose_adapters_plan_the_head_are_refused(image, how):
    st, _ = image("tiny6")
    if how == "pair":
        lora = synth.make_lora_st("tiny6", rank=8, seed=1)                 # its pairs include the head
        m = runtime.Model(st, max_batch=4, token_chunk_size=64, adapters=[(lora, 1.0)])
    else:
        m = runtime.Model(st, max_batch=4, token_chunk_size=64, adapter_places=1, adapter_targets=("head",))
    try:
        m.state.load(m.state.init(), 0)
        before = feed(m, 0, [1, 5, 9])
        with pytest.raises(capi.B200Error) as e:
            m.head_format("FP8")
        assert e.value.code == capi.ERR_UNSUPPORTED
        m.state.load(m.state.init(), 0)
        assert same_bits(feed(m, 0, [1, 5, 9]), before)
    finally:
        m.close()


def test_refusals(image):
    st, _ = image("tiny6")
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, exact=True)           # precision 1
    try:
        m.state.load(m.state.init(), 0)
        before = feed(m, 0, [1, 5, 9])
        for kind, code in (("Int8", capi.ERR_UNSUPPORTED), (3, capi.ERR_UNSUPPORTED), (7, capi.ERR_INVALID)):
            with pytest.raises(capi.B200Error) as e:
                m.head_format(kind)
            assert e.value.code == code, kind
        m.head_format("None")                                # the current format: nothing to refuse
        m.state.load(m.state.init(), 0)
        assert same_bits(feed(m, 0, [1, 5, 9]), before)
    finally:
        m.close()
    assert capi.lib().b200rwkv_head_format(None, capi.QUANT_FP8) == capi.ERR_INVALID


def test_tensor_parallel_engines_are_refused(image):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    st, _ = image("small5")
    m = runtime.Model(st, max_batch=2, token_chunk_size=16, devices=[0, 1])
    try:
        with pytest.raises(capi.B200Error) as e:
            m.head_format("Int4")
        assert e.value.code == capi.ERR_UNSUPPORTED
    finally:
        m.close()


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_step_weight_bytes(image, fmt):
    """profile_step's gemm_weight_bytes falls by the f16 head's bytes less the format's."""
    st, _ = image("small6")
    m = runtime.Model(st, max_batch=4, token_chunk_size=64)
    try:
        V, C = m.info["num_vocab"], m.info["num_emb"]
        for s in range(4):
            m.state.load(m.state.init(), s)
        _, _, f16_bytes = m.profile_step([0, 1, 2, 3], [1, 2, 3, 4])
        m.head_format(fmt)
        _, _, q_bytes = m.profile_step([0, 1, 2, 3], [1, 2, 3, 4])
        assert f16_bytes - q_bytes == 2 * V * C - H.head_bytes(V, C, FORMATS[fmt])
    finally:
        m.close()
