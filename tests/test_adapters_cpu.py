"""CPU-side checks of unblended LoRA adapters (b200rwkv_create_adapters / b200rwkv_bind_adapter / b200rwkv_op_adapter): the
ctypes bindings, the refusals the entries make before any CUDA call, and the oracle's unblended adapter path against the
load-time blend it restates (AdapterOracle, the unblended path on top of the NumPy oracle)."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, synth
from oracle import rwkv_numpy as O

from adapter_oracle import AdapterOracle


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def _opt(**kw):
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    for k, v in kw.items():
        setattr(opt, k, v)
    return opt


def _create(st, adapters, opt=None, n=None):
    """b200rwkv_create_adapters on (image, alpha) pairs; returns the status."""
    opt = opt or _opt()
    imgs = [np.ascontiguousarray(a, np.uint8) if a is not None else None for a, _ in adapters]
    k = max(len(imgs), 1)
    ptrs = (C.c_void_p * k)(*[i.ctypes.data if i is not None else None for i in imgs])
    lens = (C.c_size_t * k)(*[i.size if i is not None else 0 for i in imgs])
    alphas = (C.c_float * k)(*[float(a) for _, a in adapters])
    h = C.c_void_p()
    rc = capi.lib().b200rwkv_create_adapters(capi.ptr(st), st.size, C.byref(opt), len(imgs) if n is None else n,
                                             C.cast(ptrs, C.c_void_p), C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p),
                                             C.byref(h))
    if h:               # a call that passed every check on a machine with a GPU built an engine
        capi.lib().b200rwkv_destroy(h)
    return rc


@pytest.fixture(scope="module")
def tiny6():
    return synth.make_st("tiny6", 0)


def _pairs(preset, **tensors):
    return synth.pack_st({k: np.asarray(v, np.float16) for k, v in tensors.items()})


def test_bindings_declare_the_entries():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    P = C.c_void_p
    assert sym["b200rwkv_create_adapters"] == (C.c_int32, [P, C.c_size_t, C.POINTER(capi.Options), C.c_int32, P, P, P, C.POINTER(P)])
    assert sym["b200rwkv_bind_adapter"] == (C.c_int32, [P, C.c_int32, P, P])
    assert sym["b200rwkv_op_adapter"] == (C.c_int32, [C.c_int32] * 5 + [P] * 5)
    for name in ("b200rwkv_create_adapters", "b200rwkv_bind_adapter", "b200rwkv_op_adapter"):
        assert getattr(capi.lib(), name).argtypes == sym[name][1]


def test_create_adapters_refuses_bad_counts_and_images(tiny6):
    good = synth.make_lora_st("tiny6", rank=8, seed=1)
    for n in (0, -1, 9):
        assert _create(tiny6, [(good, 1.0)] * max(n, 1), n=n) == capi.ERR_INVALID
        assert "number of adapters must be 1..8" in _last_error()
    assert _create(tiny6, [(good, 1.0), (None, 1.0)]) == capi.ERR_INVALID
    assert "null adapter image" in _last_error()
    bad = _opt()
    bad.struct_bytes = 4
    assert _create(tiny6, [(good, 1.0)], opt=bad) == capi.ERR_INVALID


def test_create_adapters_refuses_bad_files(tiny6):
    C_, F = 256, 896
    a = np.full((C_, 8), 0.01)
    b = np.full((C_, 8), 0.01)
    # a full tensor the model has
    full = synth.pack_st({"blocks.0.att.key.weight": np.zeros((C_, C_), np.float16)})
    assert _create(tiny6, [(full, 1.0)]) == capi.ERR_UNSUPPORTED
    assert "full tensor" in _last_error()
    # a pair on something that is not a projection matrix
    odd = _pairs("tiny6", **{"blocks.0.att.time_mix_w1.lora.0": np.zeros((C_, 8)), "blocks.0.att.time_mix_w1.lora.1": np.zeros((160, 8))})
    assert _create(tiny6, [(odd, 1.0)]) == capi.ERR_UNSUPPORTED
    # a missing half, either way round
    for name in ("lora.0", "lora.1"):
        half = _pairs("tiny6", **{f"blocks.1.att.key.{name}": a})
        assert _create(tiny6, [(half, 1.0)]) == capi.ERR_INVALID, name
        assert "lora.1" in _last_error() or "lora.0" in _last_error()
    # shapes that do not match the matrix, or the two halves
    for lo0, lo1 in ((np.zeros((C_ + 8, 8)), b), (a, np.zeros((C_, 4))), (np.zeros((F, 8)), b)):
        bad = _pairs("tiny6", **{"blocks.0.att.key.lora.0": lo0, "blocks.0.att.key.lora.1": lo1})
        assert _create(tiny6, [(bad, 1.0)]) == capi.ERR_INVALID
        assert "shapes do not match" in _last_error()
    # rank 129 is one more than a tail k block holds; 128 passes the host checks (and then needs a GPU)
    r129 = _pairs("tiny6", **{"blocks.0.ffn.value.lora.0": np.zeros((F, 129)), "blocks.0.ffn.value.lora.1": np.zeros((C_, 129))})
    assert _create(tiny6, [(r129, 1.0)]) == capi.ERR_UNSUPPORTED
    assert "above 128" in _last_error()
    r128 = _pairs("tiny6", **{"blocks.0.ffn.value.lora.0": np.zeros((F, 128)), "blocks.0.ffn.value.lora.1": np.zeros((C_, 128))})
    assert _create(tiny6, [(r128, 1.0)]) not in (capi.ERR_UNSUPPORTED,)
    # an f32 pair
    f32 = synth.pack_st({"blocks.0.att.key.lora.0": np.zeros((C_, 8), np.float32), "blocks.0.att.key.lora.1": np.zeros((C_, 8), np.float32)})
    assert _create(tiny6, [(f32, 1.0)]) == capi.ERR_UNSUPPORTED
    # the second file is checked too
    assert _create(tiny6, [(synth.make_lora_st("tiny6", 8, 1), 1.0), (r129, 1.0)]) == capi.ERR_UNSUPPORTED


def test_create_adapters_refuses_devices_and_quantised_layers(tiny6):
    good = synth.make_lora_st("tiny6", rank=8, seed=1)
    two = _opt(num_devices=2)
    two.devices[0], two.devices[1] = 0, 1
    assert _create(tiny6, [(good, 1.0)], opt=two) == capi.ERR_UNSUPPORTED
    assert "one GPU" in _last_error()
    # layer 0 quantised: a pair on blocks.0 is refused, a file with pairs only on blocks.1 and the head passes the host checks
    q = _opt(quant_layers=1, quant_type=capi.QUANT_INT8)
    assert _create(tiny6, [(good, 1.0)], opt=q) == capi.ERR_UNSUPPORTED
    assert "quantised" in _last_error()
    w = O.parse_st(good)
    only1 = synth.pack_st({k: v for k, v in w.items() if not k.startswith("blocks.0.")})
    assert _create(tiny6, [(only1, 1.0)], opt=q) not in (capi.ERR_UNSUPPORTED, capi.ERR_INVALID)


def test_bind_adapter_refusals_without_an_engine():
    L = capi.lib()
    s = np.array([0, 1, 2], np.int32)
    ids = np.array([1, 0, 2], np.int32)
    assert L.b200rwkv_bind_adapter(None, 3, None, capi.ptr(ids)) == capi.ERR_INVALID
    assert L.b200rwkv_bind_adapter(None, 3, capi.ptr(s), None) == capi.ERR_INVALID
    for n in (0, -1, 1025):
        big = np.arange(max(n, 1), dtype=np.int32)
        assert L.b200rwkv_bind_adapter(None, n, capi.ptr(big), capi.ptr(big)) == capi.ERR_INVALID
        assert "nslot" in _last_error()
    neg = np.array([0, -1, 2], np.int32)
    assert L.b200rwkv_bind_adapter(None, 3, capi.ptr(neg), capi.ptr(ids)) == capi.ERR_STATE
    dup = np.array([4, 1, 4], np.int32)
    assert L.b200rwkv_bind_adapter(None, 3, capi.ptr(dup), capi.ptr(ids)) == capi.ERR_INVALID
    assert "duplicate slot" in _last_error()
    bad = np.array([1, -2, 0], np.int32)
    assert L.b200rwkv_bind_adapter(None, 3, capi.ptr(s), capi.ptr(bad)) == capi.ERR_INVALID
    assert "unknown adapter id -2" in _last_error()
    assert L.b200rwkv_bind_adapter(None, 3, capi.ptr(s), capi.ptr(ids)) == capi.ERR_INVALID
    assert "null engine" in _last_error()


def test_op_adapter_refusals_before_any_cuda_call():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((4, 64)).astype(np.float16)
    a = [rng.standard_normal((64, 8)).astype(np.float16)]
    ids = np.array([1, 0, 1, 0], np.int32)
    cases = [
        (dict(x=x, lora_a=a, ids=ids, precision=2), "precision"),
        (dict(x=rng.standard_normal((4, 60)).astype(np.float16), lora_a=[np.zeros((60, 8), np.float16)], ids=ids), "K must"),
        (dict(x=np.zeros((129, 64), np.float16), lora_a=a, ids=np.zeros(129, np.int32)), "T must"),
        (dict(x=np.zeros((2, 17, 64), np.float16), lora_a=a, ids=np.zeros(17, np.int32), precision=1), "T must"),
        (dict(x=x, lora_a=[np.zeros((64, 129), np.float16)], ids=ids), "rank"),
        (dict(x=x, lora_a=a, ids=np.array([1, 0, 2, 0], np.int32)), "adapter id"),
        (dict(x=x, lora_a=a, ids=np.array([1, 0, -1, 0], np.int32)), "adapter id"),
        (dict(x=x, lora_a=a * 9, ids=ids), "n must"),
    ]
    for kw, msg in cases:
        with pytest.raises(capi.B200Error) as ei:
            capi.op_adapter(**kw)
        assert ei.value.code == capi.ERR_INVALID and msg in str(ei.value), (msg, str(ei.value))
    L = capi.lib()
    r = np.array([8], np.int32)
    assert L.b200rwkv_op_adapter(0, 4, 64, 0, 1, capi.ptr(r), None, capi.ptr(ids), capi.ptr(x), capi.ptr(x)) == capi.ERR_INVALID


@pytest.mark.parametrize("preset", ["tiny5", "tiny6", "tiny7", "small6"])
def test_oracle_unblended_adapter_equals_the_load_time_blend(preset):
    """Binding an adapter is the unblended equivalent of blending the same file at load: the oracle's unblended path agrees
    with blend_lora + Oracle within 1e-3 with the same argmax, on one run and on a state carried between runs."""
    st = synth.make_st(preset, 0)
    w = O.parse_st(st)
    targets = ("att.receptance", "att.key", "att.value", "att.gate", "att.output", "ffn.key", "ffn.value", "ffn.receptance")
    lora = O.parse_st(synth.make_lora_st(preset, rank=16, seed=3, targets=targets))
    alpha = 0.1          # the synthetic pairs move the logits by ~20 % at this alpha
    blended = O.Oracle(O.blend_lora(w, lora, alpha), "f16")
    unblended = AdapterOracle(w, "f16", adapter=(lora, alpha))
    plain = O.Oracle(w, "f16")
    toks = [3, 17, 250, 9, 77, 1]
    want, st_b = blended.run(toks, blended.state_init(), full=True)
    got, st_u = unblended.run(toks, unblended.state_init(), full=True)
    base, _ = plain.run(toks, plain.state_init(), full=True)
    for r in range(len(toks)):
        err = np.abs(got[r] - want[r]).max() / np.abs(want[r]).max()
        assert err <= 1e-3 and got[r].argmax() == want[r].argmax(), (preset, r, err)
    assert np.abs(st_u - st_b).max() <= 1e-3 * max(1.0, np.abs(st_b).max())
    # the adapter changes the logits well beyond that tolerance, so the comparison has something to see
    assert np.abs(base - want).max() / np.abs(want).max() > 1e-2
