"""Adapter places on the GPU (b200rwkv_create_adapter_places / b200rwkv_load_adapter / b200rwkv_unload_adapter): empty places
leave the base model's bits and launches alone, a loaded place gives the bits of an engine created with the file at that id
(b200rwkv_create_adapters, same plans), a swap leaves the other places' slots alone, and every refusal changes nothing."""
import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

from adapter_oracle import AdapterOracle
from test_gpu_adapters import _run_calls

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
LAST, FULL, NONE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE
ALL = tuple(capi.TARGETS)
KINDS = tuple(t for t in ALL if t != "head")
# (rank, alpha, targets); make_lora_st pairs the head too.  Files 1-3 pair every kind between them, and so do files 1, 3, 4,
# so an engine created with either list plans every matrix, as a places engine targeting everything does.
FILES = ((8, 0.1, ("att.key", "att.value", "att.output", "ffn.key", "ffn.value")),
         (16, -0.15, ("att.receptance", "att.gate", "ffn.receptance", "ffn.value", "att.key")),
         (32, 0.12, ("att.receptance", "att.output", "ffn.key")),
         (64, -0.1, ("att.value", "att.gate", "ffn.receptance")))


def _file(preset, i):
    r, a, t = FILES[i]
    return synth.make_lora_st(preset, rank=r, seed=31 + i, targets=t), a


def _places(st, n=3, targets=ALL, S=4, chunk=64, **kw):
    return runtime.Model(st, max_batch=S, token_chunk_size=chunk, adapter_places=n, adapter_targets=targets, **kw)


def _created(st, files, S=4, chunk=64, **kw):
    return runtime.Model(st, max_batch=S, token_chunk_size=chunk, adapters=files, **kw)


def _same_bits(got, want):
    assert len(got) == len(want)
    for g, x in zip(got, want):
        assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(x).view(np.uint32))


def _calls_match(m, ref, seed, V, S=4):
    """_run_calls on both engines: the same bits, and the same launches per call mix"""
    n0, n1 = m.launch_count(), ref.launch_count()
    got, want = _run_calls(m, seed, V, S), _run_calls(ref, seed, V, S)
    assert m.launch_count() - n0 == ref.launch_count() - n1
    _same_bits(got, want)


def _check_oracle(rows, want):
    rows, want = np.asarray(rows), np.asarray(want)
    assert np.abs(rows.astype(np.float64) - want).max() / np.abs(want).max() <= REL_TOL
    assert np.array_equal(rows.argmax(-1), want.argmax(-1))


def _close(*ms):
    for m in ms:
        m.close()


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_empty_places_change_nothing_for_the_base_model(preset):
    st = synth.make_st(preset, 0)
    base = runtime.Model(st, max_batch=4, token_chunk_size=64, devices=[0])
    pl = _places(st)
    V = pl.info["num_vocab"]
    try:
        _calls_match(pl, base, 4, V)
        # a load, a bound run, an unbind and an unload later: the base model's bits again
        pl.load_adapter(2, *_file(preset, 0))
        pl.bind_adapter([0, 2], [2, 2])
        _run_calls(pl, 5, V, 4)
        pl.bind_adapter([0, 2], [0, 0])
        pl.unload_adapter(2)
        _calls_match(pl, base, 4, V)
    finally:
        _close(base, pl)


@pytest.mark.parametrize("preset,precision", [("tiny5", 0), ("tiny6", 0), ("tiny7", 0), ("small6", 0), ("tiny6", 1)])
def test_loading_equals_creation(preset, precision):
    st = synth.make_st(preset, 0)
    files = [_file(preset, i) for i in range(3)]
    ref = _created(st, files, precision=precision)
    pl = _places(st, precision=precision)
    V = pl.info["num_vocab"]
    try:
        for i in (3, 1, 2):
            pl.load_adapter(i, *files[i - 1])
        for m in (pl, ref):
            m.bind_adapter([0, 1, 2, 3], [1, 3, 0, 2])
        _calls_match(pl, ref, 7, V)
    finally:
        _close(ref, pl)


def test_swapping_one_place_leaves_the_others_alone():
    st = synth.make_st("tiny6", 0)
    f = [_file("tiny6", i) for i in range(4)]
    old, new = _created(st, f[:3]), _created(st, [f[0], f[3], f[2]])
    pl = _places(st)
    V = pl.info["num_vocab"]
    rng = np.random.default_rng(8)
    try:
        for i in (1, 2, 3):
            pl.load_adapter(i, *f[i - 1])
        for m in (pl, old):
            m.bind_adapter([0, 1, 2, 3], [1, 3, 2, 0])
            for s in range(4):
                m.state.load(m.state.init(), s)

        def step(n):
            """one call on every slot, the same on the places engine and on `old`: their rows and states agree bit for bit"""
            toks = rng.integers(1, V, size=4 * n).tolist()
            out = [m.infer_raw([0, 1, 2, 3], [n] * 4, toks, [FULL] * 4) + [m.state.back(s) for s in range(4)] for m in (pl, old)]
            _same_bits(*out)

        step(3)                                  # before
        for m in (pl, old):
            m.bind_adapter([2], [0])
        pl.unload_adapter(2)
        step(1)                                  # during: place 2 empty, slots on places 1 and 3 continue
        pl.load_adapter(2, *f[3])
        step(5)                                  # after, slot 2 still unbound
        # the swapped engine is the engine created with [f1, f4, f3]
        for m in (pl, new):
            m.bind_adapter([0, 1, 2, 3], [1, 3, 2, 0])
        _calls_match(pl, new, 9, V)
        # a slot bound to place 2 now runs the fourth file
        orc = AdapterOracle(O.parse_st(st), "f16", adapter=(O.parse_st(f[3][0]), f[3][1]))
        pl.state.load(pl.state.init(), 2)
        toks = rng.integers(1, V, size=9).tolist()
        got = pl.infer_raw([2], [9], toks, [FULL])[0]
        want, _ = orc.run(toks, orc.state_init(), full=True)
        _check_oracle(got, want)
    finally:
        _close(old, new, pl)


@pytest.mark.parametrize("preset", ["tiny6", "tiny7"])
def test_a_file_pairing_some_of_the_targets(preset):
    st = synth.make_st(preset, 0)
    part = _file(preset, 2)                     # att.receptance, att.output, ffn.key and the head
    ref = _created(st, [part, _file(preset, 0), _file(preset, 1)])
    pl = _places(st)
    V = pl.info["num_vocab"]
    try:
        pl.load_adapter(1, *part)
        for m in (pl, ref):
            m.bind_adapter([0, 3], [1, 1])
        _calls_match(pl, ref, 11, V)
        orc = AdapterOracle(O.parse_st(st), "f16", adapter=(O.parse_st(part[0]), part[1]))
        pl.state.load(pl.state.init(), 0)
        toks = np.random.default_rng(12).integers(1, V, size=12).tolist()
        got = pl.infer_raw([0], [12], toks, [FULL])[0]
        want, _ = orc.run(toks, orc.state_init(), full=True)
        _check_oracle(got, want)
    finally:
        _close(ref, pl)


def test_head_rank_changes_reach_the_snapshot_head():
    """A bound slot's head rank goes 8 -> none -> 64, with the snapshot launches set up while the place is empty: snapshot
    rows of tokens without an output row (their own head launch and shrink) equal the FULL rows of the same tokens."""
    st = synth.make_st("tiny6", 0)
    r8 = synth.make_lora_st("tiny6", rank=8, seed=51, targets=("att.key",))
    r64 = synth.make_lora_st("tiny6", rank=64, seed=52, targets=("att.key",))
    fill = synth.make_lora_st("tiny6", rank=8, seed=53, targets=KINDS)          # the other place: every kind
    ref = _created(st, [(r64, 0.3), (fill, 0.1)])
    pl = _places(st, n=2)
    V = pl.info["num_vocab"]
    rng = np.random.default_rng(13)
    try:
        pl.load_adapter(2, fill, 0.1)
        pl.load_adapter(1, r8, 0.3)
        pl.bind_adapter([0], [1])
        pl.infer_raw([0], [6], rng.integers(1, V, size=6).tolist(), [LAST])
        pl.bind_adapter([0], [0])
        pl.unload_adapter(1)
        # snapshots between the loads (on an unbound slot): the snapshot launches are made now
        pl.infer_snapshots([1], [5], rng.integers(1, V, size=5).tolist(), [NONE], [(0, 2), (0, 5)])
        pl.load_adapter(1, r64, 0.3)
        for m in (pl, ref):
            m.bind_adapter([0], [1])
            m.state.load(m.state.init(), 0)
        toks = rng.integers(1, V, size=20).tolist()
        at = (3, 10, 20)
        _, _, snaps = pl.infer_snapshots([0], [20], toks, [LAST], [(0, p) for p in at])
        ids, probs = pl.sample_topk([0], top_k=8)
        ref.infer_raw([0], [20], toks, [LAST])
        ref_ids, ref_probs = ref.sample_topk([0], top_k=8)
        assert np.array_equal(ids, ref_ids) and np.array_equal(probs.view(np.uint32), ref_probs.view(np.uint32))
        pl.state.load(pl.state.init(), 0)
        full = pl.infer_raw([0], [20], toks, [FULL])[0]
        for p, sn in zip(at, snaps):
            _, row = pl.state.snapshot_back(sn, with_logits=True)
            assert np.array_equal(row.view(np.uint32), full[p - 1].view(np.uint32)), p
    finally:
        _close(ref, pl)


def test_unload_and_reload_on_a_created_engine():
    st = synth.make_st("tiny6", 0)
    f = [_file("tiny6", i) for i in range(4)]
    ca, new = _created(st, f[:3]), _created(st, [f[0], f[3], f[2]])
    V = ca.info["num_vocab"]
    try:
        ca.unload_adapter(2)
        ca.load_adapter(2, *f[3])
        for m in (ca, new):
            m.bind_adapter([0, 1, 2, 3], [2, 1, 3, 2])
        _calls_match(ca, new, 14, V)
    finally:
        _close(ca, new)


def _refused(fn, code, fragment):
    with pytest.raises(capi.B200Error) as ei:
        fn()
    assert ei.value.code == code and fragment in str(ei.value), str(ei.value)


def test_refusals_on_a_live_engine_change_nothing():
    st = synth.make_st("tiny6", 0)
    w = O.parse_st(st)
    C_, F = w["blocks.0.att.key.weight"].shape[1], w["blocks.0.ffn.key.weight"].shape[0]
    pl = _places(st, n=2, targets=("att.key", "att.value", "ffn.key", "head"))
    good = synth.make_lora_st("tiny6", rank=8, seed=61, targets=("att.key", "ffn.key"))
    pl.load_adapter(1, good, 0.2)
    pl.bind_adapter([0, 2], [1, 1])
    V = pl.info["num_vocab"]

    def pairs(name, a, b):
        return synth.pack_st({f"{name}.lora.0": np.zeros(a, np.float16), f"{name}.lora.1": np.zeros(b, np.float16)})

    try:
        want = _run_calls(pl, 15, V, 4)
        _refused(lambda: pl.load_adapter(1, good, 0.2), capi.ERR_STATE, "place 1 holds an adapter")
        _refused(lambda: pl.unload_adapter(1), capi.ERR_STATE, "slot 0 is bound")
        _refused(lambda: pl.unload_adapter(2), capi.ERR_STATE, "place 2 is empty")
        _refused(lambda: pl.bind_adapter([1], [2]), capi.ERR_STATE, "place 2 is empty")
        _refused(lambda: pl.load_adapter(3, good, 0.2), capi.ERR_INVALID, "outside 1..n")
        # att.output is not among the targets
        outside = synth.make_lora_st("tiny6", rank=8, seed=62, targets=("att.key", "att.output"))
        _refused(lambda: pl.load_adapter(2, outside, 0.2), capi.ERR_UNSUPPORTED, "blocks.0.att.output")
        _refused(lambda: pl.load_adapter(2, pairs("blocks.1.ffn.key", (C_, 129), (F, 129)), 1.0), capi.ERR_UNSUPPORTED,
                 "above 128")
        _refused(lambda: pl.load_adapter(2, pairs("blocks.1.att.key", (C_ + 8, 8), (C_, 8)), 1.0), capi.ERR_INVALID,
                 "shapes do not match")
        _same_bits(_run_calls(pl, 15, V, 4), want)
    finally:
        pl.close()
    # a pair on a matrix of a quantised layer (layer 0 holds Int8 matrices, so only layers 1.. and the head are planned)
    pq = _places(st, n=2, quant=1, quant_type="Int8")
    try:
        keys = O.parse_st(synth.make_lora_st("tiny6", rank=8, seed=63, targets=("att.key",)))
        pq.load_adapter(1, synth.pack_st({k: v for k, v in keys.items() if not k.startswith("blocks.0.")}), 0.2)
        pq.bind_adapter([1], [1])
        want = _run_calls(pq, 16, V, 4)
        _refused(lambda: pq.load_adapter(2, pairs("blocks.0.att.key", (C_, 8), (C_, 8)), 1.0), capi.ERR_UNSUPPORTED,
                 "quantised")
        _same_bits(_run_calls(pq, 16, V, 4), want)
    finally:
        pq.close()
