"""CPU-side checks of adapter places (b200rwkv_create_adapter_places / b200rwkv_load_adapter / b200rwkv_unload_adapter): the
ctypes bindings and every refusal the entries make before any CUDA call or without an engine."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, synth

ALL = (1 << 9) - 1


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def _opt(**kw):
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    for k, v in kw.items():
        setattr(opt, k, v)
    return opt


def _create(st, n, targets, opt=None, out=True):
    """b200rwkv_create_adapter_places; returns the status."""
    opt = _opt() if opt is None else opt
    h = C.c_void_p()
    rc = capi.lib().b200rwkv_create_adapter_places(capi.ptr(st), st.size, opt, n, targets, C.byref(h) if out else None)
    if h:               # a call that passed every check on a machine with a GPU built an engine
        capi.lib().b200rwkv_destroy(h)
    return rc


@pytest.fixture(scope="module")
def tiny6():
    return synth.make_st("tiny6", 0)


@pytest.fixture(scope="module")
def tiny7():
    return synth.make_st("tiny7", 0)


def test_bindings_declare_the_entries():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    P = C.c_void_p
    assert sym["b200rwkv_create_adapter_places"] == (C.c_int32, [P, C.c_size_t, C.POINTER(capi.Options), C.c_int32, C.c_uint32,
                                                                 C.POINTER(P)])
    assert sym["b200rwkv_load_adapter"] == (C.c_int32, [P, C.c_int32, P, C.c_size_t, C.c_float])
    assert sym["b200rwkv_unload_adapter"] == (C.c_int32, [P, C.c_int32])
    for name in ("b200rwkv_create_adapter_places", "b200rwkv_load_adapter", "b200rwkv_unload_adapter"):
        assert getattr(capi.lib(), name).argtypes == sym[name][1]
    # the target bits, one per kind of matrix, in the header's order
    assert sorted(capi.TARGETS.values()) == [1 << i for i in range(9)]
    assert capi.TARGETS["head"] == capi.TARGET_HEAD == 1 << 8


def test_create_refuses_bad_counts_targets_and_options(tiny6):
    for n in (0, -1, 9):
        assert _create(tiny6, n, ALL) == capi.ERR_INVALID
        assert "number of adapter places must be 1..8" in _last_error()
    for targets in (0, 1 << 9, ALL | (1 << 31)):
        assert _create(tiny6, 2, targets) == capi.ERR_INVALID
        assert "B200RWKV_TARGET_" in _last_error()
    assert _create(tiny6, 2, ALL, out=False) == capi.ERR_INVALID
    assert "null argument" in _last_error()
    h = C.c_void_p()
    assert capi.lib().b200rwkv_create_adapter_places(capi.ptr(tiny6), tiny6.size, None, 2, ALL, C.byref(h)) == capi.ERR_INVALID
    assert "null argument" in _last_error()
    bad = _opt()
    bad.struct_bytes = 4
    assert _create(tiny6, 2, ALL, opt=bad) == capi.ERR_INVALID
    assert "struct_bytes" in _last_error()


def test_create_refuses_two_devices_and_targets_without_an_f16_matrix(tiny6, tiny7):
    two = _opt(num_devices=2)
    two.devices[0], two.devices[1] = 0, 1
    assert _create(tiny6, 2, ALL, opt=two) == capi.ERR_UNSUPPORTED
    assert "one GPU" in _last_error()
    # v7 has no att.gate / ffn.receptance matrix: those bits alone name nothing
    assert _create(tiny7, 2, capi.TARGET_ATT_G | capi.TARGET_FFN_R) == capi.ERR_UNSUPPORTED
    assert "name no f16 projection matrix" in _last_error()
    # every layer quantised: only the head is left in f16
    L = synth.PRESETS["tiny6"].L
    q = _opt(quant_layers=L, quant_type=capi.QUANT_INT8)
    assert _create(tiny6, 2, capi.TARGET_ATT_K | capi.TARGET_FFN_V, opt=q) == capi.ERR_UNSUPPORTED
    assert "name no f16 projection matrix" in _last_error()
    assert _create(tiny6, 2, capi.TARGET_HEAD, opt=q) not in (capi.ERR_UNSUPPORTED, capi.ERR_INVALID)


def test_a_well_formed_create_passes_the_host_checks(tiny6, tiny7):
    """Without a GPU a well-formed create ends at the device check (there is no CPU fallback); with one it builds."""
    for st, n, targets in ((tiny6, 8, ALL), (tiny7, 1, capi.TARGET_ATT_G | capi.TARGET_ATT_K)):
        rc = _create(st, n, targets)      # v7: the ATT_G bit is skipped, ATT_K names matrices
        assert rc in (capi.OK, capi.ERR_CUDA), _last_error()
        if rc == capi.ERR_CUDA:
            assert "no CPU fallback" in _last_error()


def test_load_and_unload_refusals_without_an_engine():
    L = capi.lib()
    img = synth.make_lora_st("tiny6", rank=8, seed=1)
    for id_ in (0, -1):
        assert L.b200rwkv_load_adapter(None, id_, capi.ptr(img), img.size, 1.0) == capi.ERR_INVALID
        assert f"id {id_} outside 1..n" in _last_error()
        assert L.b200rwkv_unload_adapter(None, id_) == capi.ERR_INVALID
        assert f"id {id_} outside 1..n" in _last_error()
    assert L.b200rwkv_load_adapter(None, 1, None, img.size, 1.0) == capi.ERR_INVALID
    assert "null adapter image" in _last_error()
    assert L.b200rwkv_load_adapter(None, 1, capi.ptr(img), 4, 1.0) == capi.ERR_INVALID
    assert "null adapter image" in _last_error()
    assert L.b200rwkv_load_adapter(None, 1, capi.ptr(img), img.size, 1.0) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    assert L.b200rwkv_unload_adapter(None, 1) == capi.ERR_INVALID
    assert "null engine" in _last_error()
