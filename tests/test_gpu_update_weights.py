"""GPU tests of the in-place weight updates (b200rwkv_update_weights, b200rwkv_update_weights_device), all bit-exact: an engine
created from image X, run (graphs captured), then updated to Y, against an engine created from Y, on a mixed workload of
LAST / FULL / NONE / SCORE entries with score_top, a snapshot, pooled hidden rows, sample_topk / sample_probs and states,
with equal launch counts -- for every model version, both precisions, state-tuned models, the four quantised formats on part
and all of the model, batch-invariant engines, bound adapters, adapter places and adapters on quantised layers.  Partial
images against creation from the merged image; a round trip; what an update leaves alone; the device path against the host
path with F16-rounded values; and every refusal, after which the engine computes what one that never saw it computes."""
import dataclasses
import json
import struct

import numpy as np
import pytest
import torch

from ai00_server_b200 import capi, runtime, synth
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

S = 4
LAST, FULL, NONE, SCORE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_SCORE


def _shape(preset, **kw):
    return dataclasses.replace(synth.PRESETS[preset], **kw)


def _tensors(st):
    return {k: np.array(v) for k, v in O.parse_st(st).items()}


def _merged(x, y, names):
    t = _tensors(x)
    yt = _tensors(y)
    for n in names:
        t[n] = yt[n]
    return synth.pack_st(t)


def _partial(y, names):
    yt = _tensors(y)
    return synth.pack_st({n: yt[n] for n in names})


def _image(entries):
    """safetensors image of {name: (dtype string, shape, raw bytes)}, any dtype"""
    header, off, blobs = {}, 0, []
    for name, (dt, shape, raw) in entries.items():
        header[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + len(raw)]}
        blobs.append(raw)
        off += len(raw)
    h = json.dumps(header).encode()
    h += b" " * ((-len(h)) % 8)
    return np.frombuffer(struct.pack("<Q", len(h)) + h + b"".join(blobs), np.uint8).copy()


def _work(m, seed):
    """The mixed workload: every output as arrays, and the launches it made"""
    V, L = m.info["num_vocab"], m.info["num_layer"]
    rng = np.random.default_rng(seed)
    n0 = m.launch_count()
    out = []
    m.keep_hidden_pooled([0, L - 1], "mean")
    for s in range(S):
        m.state.load(m.state.init(), s)
    out += m.infer_raw(list(range(S)), [1] * S, rng.integers(1, V, size=S).tolist(), [LAST] * S)
    lens = [5, 0, 40, 2]
    out += m.infer_raw([3, 1, 0, 2], lens, rng.integers(1, V, size=sum(lens)).tolist(), [FULL, LAST, NONE, LAST])
    out += [m.last_hidden_pooled(0)[0].copy(), m.last_hidden_pooled(L - 1)[0].copy()]
    rows, scores, tops = m.infer_ex([0, 1], [6, 3], rng.integers(1, V, size=9).tolist(), [SCORE, FULL], top_n=4)
    out += rows + [scores[0][0], scores[0][1].view(np.float32), tops[0][0].view(np.float32), tops[0][1]]
    rows, _, snaps = m.infer_snapshots([2, 3], [7, 1], rng.integers(1, V, size=8).tolist(), [LAST, LAST], at=[(0, 3)])
    st, lg = m.state.snapshot_back(snaps[0], with_logits=True)
    snaps[0].free()
    out += rows + [st, lg]
    ids, p = m.sample_topk(list(range(S)), top_k=8)
    out += [ids.view(np.float32), p, m.sample_probs([0, 1])]
    out += [m.state.back(s) for s in range(S)] + [m.state.init()]
    m.keep_hidden_pooled([])
    return out, m.launch_count() - n0


def _same(a, b):
    (ga, na), (gb, nb) = a, b
    assert na == nb
    assert len(ga) == len(gb)
    for x, y in zip(ga, gb):
        assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))


def _model(st, setup=None, **kw):
    m = runtime.Model(st, max_batch=S, token_chunk_size=64, **kw)
    if setup:
        setup(m)
    return m


def _update_equals_creation(x, y, update, setup=None, **kw):
    """A from x, worked, updated by update(A); B from y: the same bits and launches"""
    a = _model(x, setup, **kw)
    try:
        _work(a, 1)
        update(a)
        b = _model(y, setup, **kw)
        try:
            _same(_work(a, 2), _work(b, 2))
        finally:
            b.close()
    finally:
        a.close()


def _bind(m):
    m.bind_adapter([0, 2], [1, 2])


def _place(file):
    def setup(m):
        m.load_adapter(1, *file)
        m.bind_adapter([1, 3], [1, 1])
    return setup


def _adapter_files(preset):
    return [(synth.make_lora_st(preset, rank=8, seed=41), 0.1), (synth.make_lora_st(preset, rank=16, seed=42, targets=("att.key", "ffn.value")), -0.15)]


ALL_Q = [capi.QUANT_INT8, capi.QUANT_NF4, capi.QUANT_FP8, capi.QUANT_INT4]
CASES = ([(p, dict(precision=pr), None) for p in ("tiny5", "tiny6", "tiny7", "small6") for pr in (0, 1)] +
         [("tiny6ts", {}, None)] +
         [("tiny6", dict(quant=q, quant_type=qt), None) for qt in ALL_Q for q in (1, 2)] +
         [("tiny7", dict(batch_invariant=True), None),
          ("tiny6", dict(adapters=_adapter_files("tiny6")), _bind),
          ("tiny7", dict(adapter_places=2, adapter_targets=tuple(capi.TARGETS)), "place")] +
         [("tiny6", dict(quant=2, quant_type=qt, quant_adapters=True, adapters=_adapter_files("tiny6")), _bind)
          for qt in (capi.QUANT_FP8, capi.QUANT_INT4)])


def _images(preset):
    if preset == "tiny6ts":
        s = _shape("tiny6", time_state=True)
        return synth.make_st(s, 0), synth.make_st(s, 1)
    return synth.make_st(preset, 0), synth.make_st(preset, 1)


@pytest.mark.parametrize("preset,kw,setup", CASES, ids=[f"{p}-{'-'.join(f'{k}={v}' for k, v in kw.items() if k != 'adapters')}"
                                                        + ("-adapters" if "adapters" in kw else "") for p, kw, _ in CASES])
def test_update_equals_creation(preset, kw, setup):
    x, y = _images(preset)
    if setup == "place":
        setup = _place((synth.make_lora_st(preset, rank=8, seed=43), 0.2))
    _update_equals_creation(x, y, lambda m: m.update_weights(y), setup, **kw)


PARTIAL = [
    ("tiny6", ["blocks.1.att.key.weight"], {}),
    ("tiny6", ["head.weight"], {}),
    ("tiny7", ["emb.weight", "blocks.0.ln0.weight", "blocks.0.ln0.bias"], {}),
    ("tiny5", ["blocks.1.att.time_decay"], {}),
    ("tiny6", ["blocks.0.att.time_decay_w2"], {}),
    # split-K (two K slices at this shape), each slice's codes scaled by its whole row's absmax
    ("tiny6", ["blocks.1.att.output.weight"], dict(quant=2, quant_type=capi.QUANT_FP8)),
    ("tiny6", ["blocks.1.ffn.value.weight"], dict(quant=2, quant_type=capi.QUANT_INT4)),
]


@pytest.mark.parametrize("preset,names,kw", PARTIAL, ids=[f"{p}-{n[0]}" for p, n, _ in PARTIAL])
def test_partial_image_equals_creation_from_the_merged_image(preset, names, kw):
    x, y = _images(preset)
    _update_equals_creation(x, _merged(x, y, names), lambda m: m.update_weights(_partial(y, names)), **kw)


def test_time_state_only_changes_init_and_leaves_live_slots_alone():
    x, y = _images("tiny6ts")
    L = synth.PRESETS["tiny6"].L
    names = [f"blocks.{l}.att.time_state" for l in range(L)]
    a = _model(x)
    b = _model(_merged(x, y, names))
    try:
        _work(a, 1)
        before = [a.state.back(s) for s in range(S)]
        a.update_weights(_partial(y, names))
        for s in range(S):
            assert np.array_equal(a.state.back(s).view(np.uint32), before[s].view(np.uint32))
        assert np.array_equal(a.state.init(), b.state.init())
        assert not np.array_equal(a.state.init(), _model_init(x))
        _same(_work(a, 2), _work(b, 2))
    finally:
        a.close()
        b.close()


def _model_init(st):
    m = _model(st)
    try:
        return m.state.init()
    finally:
        m.close()


@pytest.mark.parametrize("kw", [{}, dict(quant=2, quant_type=capi.QUANT_FP8)], ids=["f16", "fp8"])
def test_round_trip_gives_the_original_bits(kw):
    x, y = _images("tiny7")
    a = _model(x, **kw)
    b = _model(x, **kw)
    try:
        want = _work(b, 3)
        _work(a, 1)
        a.update_weights(y)
        _work(a, 2)
        a.update_weights(x)
        _same(_work(a, 3), want)
    finally:
        a.close()
        b.close()


def test_states_snapshots_and_kept_rows_are_left_alone():
    x, y = _images("tiny6")
    m = _model(x, adapters=_adapter_files("tiny6"))
    try:
        V = m.info["num_vocab"]
        _bind(m)
        for s in range(S):
            m.state.load(m.state.init(), s)
        m.infer_raw(list(range(S)), [3] * S, list(np.arange(1, 3 * S + 1) % V), [LAST] * S)
        _, _, snaps = m.infer_snapshots([1], [4], [5, 6, 7, 8], [LAST], at=[(0, 2)])
        read = m.state.read(2)

        def look():
            ids, p = m.sample_topk(list(range(S)), top_k=8)
            return ([m.state.back(s) for s in range(S)] + list(m.state.snapshot_back(snaps[0], with_logits=True)) +
                    [m.state.snapshot_back(read), ids.view(np.float32), p, m.sample_probs(list(range(S)))])

        before = look()
        m.update_weights(y)
        after = look()
        for u, v in zip(before, after):
            assert np.array_equal(np.asarray(u).view(np.uint32), np.asarray(v).view(np.uint32))
        snaps[0].free()
        read.free()
    finally:
        m.close()


def _rounding_cases(a, i):
    """a's values in F16, BF16 or F32 by index, the F32 ones moved off the F16 grid (ties included), the BF16 ones with some
    values below F16's normal range"""
    kind = i % 3
    f = a.astype(np.float32)
    if kind == 0:
        return torch.from_numpy(a.copy()).cuda()
    if kind == 1:
        g = f.copy().reshape(-1)
        g[::7] = np.float32(3.1e-6)
        g[1::11] = np.float32(-7.7e-7)
        return torch.from_numpy(g.reshape(f.shape)).to(torch.bfloat16).cuda()
    ulp = np.abs(np.spacing(a.astype(np.float16))).astype(np.float32)
    g = f + ulp * np.float32(0.5)                   # exact ties between two F16 values
    g.reshape(-1)[::3] += ulp.reshape(-1)[::3] * np.float32(0.26)
    return torch.from_numpy(g).cuda()


def test_device_path_equals_the_host_path_with_rounded_values():
    x, y = _images("tiny6ts")
    yt = _tensors(y)
    dev = {n: _rounding_cases(v, i) for i, (n, v) in enumerate(yt.items())}
    host = {}
    for n, t in dev.items():
        if n.endswith("time_state"):
            host[n] = t.float().cpu().numpy()                   # read as f32, as creation reads it
        else:
            host[n] = t.to(torch.float16).cpu().numpy()         # round to nearest even
    assert any(t.dtype == torch.float32 and not torch.equal(t, t.half().float()) for t in dev.values())
    a = _model(x)
    b = _model(x)
    try:
        _work(a, 1)
        _work(b, 1)
        a.update_weights_from_tensors(dev)
        b.update_weights(synth.pack_st(host))
        _same(_work(a, 2), _work(b, 2))
    finally:
        a.close()
        b.close()


def _code(fn):
    try:
        fn()
    except capi.B200Error as e:
        return e.code
    return capi.OK


def test_refusals_change_nothing():
    x, y = _images("tiny6")
    ref = _model(x)
    m = _model(x)
    try:
        want = _work(ref, 2)
        _work(m, 1)
        head = _tensors(y)["head.weight"]
        key = "blocks.1.att.key.weight"
        kw_ = _tensors(y)[key]
        assert _code(lambda: m.update_weights(synth.pack_st({"blocks.9.att.key.weight": kw_}))) == capi.ERR_INVALID
        assert _code(lambda: m.update_weights(synth.pack_st({"head.weight": head[:-8]}))) == capi.ERR_INVALID
        # a known tensor first, then the refused one: nothing is written
        assert _code(lambda: m.update_weights(synth.pack_st({key: kw_, "head.weight": head.T.copy()}))) == capi.ERR_INVALID
        bf16 = (kw_.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        assert _code(lambda: m.update_weights(_image({key: ("BF16", kw_.shape, bf16.tobytes())}))) == capi.ERR_UNSUPPORTED
        assert _code(lambda: m.update_weights(synth.pack_st({key: kw_.astype(np.float32)}))) == capi.ERR_UNSUPPORTED
        assert _code(lambda: m.update_weights(np.zeros(32, np.uint8))) == capi.ERR_INVALID
        t = torch.from_numpy(kw_.copy()).cuda()
        L = capi.lib()
        table = (capi.WeightSrc * 2)()
        for i in range(2):
            table[i].name, table[i].dtype, table[i].data = key.encode(), capi.DTYPE_F16, t.data_ptr()
        assert L.b200rwkv_update_weights_device(m._h, 2, table) == capi.ERR_INVALID          # listed twice
        assert b"twice" in L.b200rwkv_last_error(None)
        host = np.ascontiguousarray(kw_)
        table[0].data = host.ctypes.data                                                    # not device memory
        assert L.b200rwkv_update_weights_device(m._h, 1, table) == capi.ERR_INVALID
        table[0].data, table[0].dtype = t.data_ptr(), 7
        assert L.b200rwkv_update_weights_device(m._h, 1, table) == capi.ERR_INVALID
        table[0].dtype, table[0].name = capi.DTYPE_F16, b"blocks.1.att.nothing"
        assert L.b200rwkv_update_weights_device(m._h, 1, table) == capi.ERR_INVALID
        assert L.b200rwkv_update_weights_device(m._h, 0, table) == capi.ERR_INVALID
        _same(_work(m, 2), want)
    finally:
        m.close()
        ref.close()


def test_lora_and_tensor_parallel_engines_are_refused():
    x, y = _images("tiny6")
    lora = _model(x, lora=[(synth.make_lora_st("tiny6", rank=8, seed=5), 0.5)])
    try:
        assert _code(lambda: lora.update_weights(y)) == capi.ERR_UNSUPPORTED
        t = torch.from_numpy(_tensors(y)["head.weight"].copy()).cuda()
        assert _code(lambda: lora.update_weights_from_tensors({"head.weight": t})) == capi.ERR_UNSUPPORTED
    finally:
        lora.close()
    # one rank of a two-rank world (b200rwkv_create_tp); the in-process front end's ranks have the same world
    tp = runtime.Model(x, max_batch=S, token_chunk_size=64, rank=0, world=2)
    try:
        assert _code(lambda: tp.update_weights(y)) == capi.ERR_UNSUPPORTED
    finally:
        tp.close()
