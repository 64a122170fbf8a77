"""CPU-side checks of per-layer hidden-state recording (b200rwkv_keep_hidden_layers / b200rwkv_last_hidden_layer): the ctypes
bindings, the refusals the two entries make before touching a device, and the bookkeeping of Model.keep_hidden(layers=...)
and Model.embed with the library stubbed out."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_bindings_declare_both_entries():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert sym["b200rwkv_keep_hidden_layers"] == (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p])
    assert sym["b200rwkv_last_hidden_layer"] == (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t])
    L = capi.lib()
    assert L.b200rwkv_keep_hidden_layers.argtypes == sym["b200rwkv_keep_hidden_layers"][1]
    assert L.b200rwkv_last_hidden_layer.argtypes == sym["b200rwkv_last_hidden_layer"][1]


def test_keep_hidden_layers_refusals_without_an_engine():
    """n outside [0, 8], a NULL layer list, a negative or repeated layer and a NULL engine are refused with ERR_INVALID
    before any CUDA call (the upper bound of a layer needs the model, so it is checked on the GPU)."""
    L = capi.lib()
    ok = np.array([0, 1, 2], np.int32)
    for n in (-1, 9, 100):
        big = np.arange(max(n, 1), dtype=np.int32)
        assert L.b200rwkv_keep_hidden_layers(None, n, capi.ptr(big)) == capi.ERR_INVALID
        assert "n must be in [0, 8]" in _last_error()
    assert L.b200rwkv_keep_hidden_layers(None, 2, None) == capi.ERR_INVALID
    assert "null layers" in _last_error()
    neg = np.array([1, -1], np.int32)
    assert L.b200rwkv_keep_hidden_layers(None, 2, capi.ptr(neg)) == capi.ERR_INVALID
    assert "negative layer -1" in _last_error()
    dup = np.array([3, 0, 3], np.int32)
    assert L.b200rwkv_keep_hidden_layers(None, 3, capi.ptr(dup)) == capi.ERR_INVALID
    assert "layer 3 is listed twice" in _last_error()
    assert L.b200rwkv_keep_hidden_layers(None, 3, capi.ptr(ok)) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    assert L.b200rwkv_keep_hidden_layers(None, 0, None) == capi.ERR_INVALID       # n = 0 (off) still needs an engine
    assert "null engine" in _last_error()
    eight = np.arange(8, dtype=np.int32)
    assert L.b200rwkv_keep_hidden_layers(None, 8, capi.ptr(eight)) == capi.ERR_INVALID
    assert "null engine" in _last_error()                   # 8 distinct layers pass the argument checks


def test_last_hidden_layer_refusals_without_an_engine():
    L = capi.lib()
    buf = np.zeros(16, np.float32)
    assert L.b200rwkv_last_hidden_layer(None, -2, capi.ptr(buf), buf.size) == capi.ERR_INVALID
    assert "negative layer -2" in _last_error()
    assert L.b200rwkv_last_hidden_layer(None, 0, capi.ptr(buf), buf.size) == capi.ERR_INVALID
    assert "null argument" in _last_error()
    assert L.b200rwkv_last_hidden_layer(None, 0, None, 0) == capi.ERR_INVALID
    assert "null argument" in _last_error()


class _FakeLib:
    """Records the arguments of the hidden-state entries; last_hidden_layer writes row r as the constant r."""

    def __init__(self, C_=4):
        self.calls, self.C = [], C_

    def b200rwkv_keep_hidden(self, h, enable):
        self.calls.append(("keep_hidden", enable))
        return 0

    def b200rwkv_keep_hidden_layers(self, h, n, p):
        layers = [] if n == 0 else np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int32)), (n,)).tolist()
        self.calls.append(("keep_hidden_layers", n, layers))
        return 0

    def b200rwkv_last_hidden_layer(self, h, layer, p, cap):
        rows = 3
        out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), (cap,))
        out[:rows * self.C] = np.repeat(np.arange(rows, dtype=np.float32) + 10 * layer, self.C)
        self.calls.append(("last_hidden_layer", layer, cap))
        return rows


class _StubModel(runtime.Model):
    def __init__(self):
        self._h = None
        self.info = {"num_emb": 4, "num_vocab": 8}
        self.infers = []

    def infer_raw(self, slots, ntok, tokens, options, out=None, keep_on_device=False):
        self.infers.append((list(slots), list(ntok), list(tokens), list(options)))
        return [np.zeros((0, 8), np.float32)]


@pytest.fixture
def fake():
    real, f = capi._lib, _FakeLib()
    capi._lib = f
    yield f
    capi._lib = real


def test_keep_hidden_keeps_the_bool_form_and_adds_layers(fake):
    m = _StubModel()
    m.keep_hidden(True)
    m.keep_hidden(False)
    m.keep_hidden(layers=[5, 0, 2])
    m.keep_hidden(layers=[])
    assert fake.calls == [("keep_hidden", 1), ("keep_hidden", 0), ("keep_hidden_layers", 3, [5, 0, 2]), ("keep_hidden_layers", 0, [])]
    got = m.last_hidden(max_rows=5, layer=2)
    assert fake.calls[-1] == ("last_hidden_layer", 2, 5 * 4)
    assert got.shape == (3, 4) and got[:, 0].tolist() == [20, 21, 22]


def test_embed_returns_the_last_row_of_one_none_call(fake):
    m = _StubModel()
    e = m.embed(3, [7, 8, 9], layer=1)
    assert m.infers == [([3], [3], [7, 8, 9], [capi.OPTION_NONE])]
    assert fake.calls == [("keep_hidden_layers", 1, [1]), ("last_hidden_layer", 1, 3 * 4), ("keep_hidden_layers", 0, [])]
    assert e.shape == (4,) and (e == 12).all()
    with pytest.raises(capi.B200Error):
        m.embed(0, [], layer=0)
