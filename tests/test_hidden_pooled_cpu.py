"""CPU-side checks of pooled hidden rows (b200rwkv_keep_hidden_pooled / b200rwkv_last_hidden_pooled): the ctypes bindings,
the refusals the two entries make before touching a device, and the bookkeeping of Model.keep_hidden_pooled,
Model.last_hidden_pooled and Model.embed_many with the library stubbed out."""
import ctypes as C
import pathlib
import re

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime

HEADER = pathlib.Path(__file__).resolve().parent.parent / "include" / "b200rwkv.h"


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_bindings_declare_both_entries():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert sym["b200rwkv_keep_hidden_pooled"] == (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32])
    assert sym["b200rwkv_last_hidden_pooled"] == (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p])
    L = capi.lib()
    assert L.b200rwkv_keep_hidden_pooled.argtypes == sym["b200rwkv_keep_hidden_pooled"][1]
    assert L.b200rwkv_last_hidden_pooled.argtypes == sym["b200rwkv_last_hidden_pooled"][1]


def test_mode_constants_match_the_header():
    text = HEADER.read_text()
    for name, value in (("POOL_LAST", capi.POOL_LAST), ("POOL_MEAN", capi.POOL_MEAN)):
        m = re.search(rf"#define\s+B200RWKV_{name}\s+(\d+)", text)
        assert m and int(m.group(1)) == value, name


def test_keep_hidden_pooled_refusals_without_an_engine():
    """n outside [0, 8], a NULL layer list, an unknown mode, a negative or repeated layer and a NULL engine are refused with
    ERR_INVALID before any CUDA call (the upper bound of a layer needs the model, so it is checked on the GPU)."""
    L = capi.lib()
    ok = np.array([0, 1, 2], np.int32)
    for n in (-1, 9, 100):
        big = np.arange(max(n, 1), dtype=np.int32)
        assert L.b200rwkv_keep_hidden_pooled(None, n, capi.ptr(big), capi.POOL_LAST) == capi.ERR_INVALID
        assert "n must be in [0, 8]" in _last_error()
    assert L.b200rwkv_keep_hidden_pooled(None, 2, None, capi.POOL_MEAN) == capi.ERR_INVALID
    assert "null layers" in _last_error()
    for mode in (-1, 2, 7):
        assert L.b200rwkv_keep_hidden_pooled(None, 3, capi.ptr(ok), mode) == capi.ERR_INVALID
        assert f"unknown mode {mode}" in _last_error()
    neg = np.array([1, -1], np.int32)
    assert L.b200rwkv_keep_hidden_pooled(None, 2, capi.ptr(neg), capi.POOL_LAST) == capi.ERR_INVALID
    assert "negative layer -1" in _last_error()
    dup = np.array([3, 0, 3], np.int32)
    assert L.b200rwkv_keep_hidden_pooled(None, 3, capi.ptr(dup), capi.POOL_MEAN) == capi.ERR_INVALID
    assert "layer 3 is listed twice" in _last_error()
    for mode in (capi.POOL_LAST, capi.POOL_MEAN):          # both modes and 8 distinct layers pass the argument checks
        eight = np.arange(8, dtype=np.int32)
        assert L.b200rwkv_keep_hidden_pooled(None, 8, capi.ptr(eight), mode) == capi.ERR_INVALID
        assert "null engine" in _last_error()
    assert L.b200rwkv_keep_hidden_pooled(None, 0, None, capi.POOL_LAST) == capi.ERR_INVALID      # n = 0 (off) still needs an engine
    assert "null engine" in _last_error()


def test_last_hidden_pooled_refusals_without_an_engine():
    L = capi.lib()
    buf = np.zeros(16, np.float32)
    ntok = np.zeros(4, np.int32)
    assert L.b200rwkv_last_hidden_pooled(None, -2, capi.ptr(buf), buf.size, capi.ptr(ntok)) == capi.ERR_INVALID
    assert "negative layer -2" in _last_error()
    assert L.b200rwkv_last_hidden_pooled(None, 0, capi.ptr(buf), buf.size, None) == capi.ERR_INVALID
    assert "null argument" in _last_error()
    assert L.b200rwkv_last_hidden_pooled(None, 0, None, 0, capi.ptr(ntok)) == capi.ERR_INVALID       # NULL out
    assert "null argument" in _last_error()


class _FakeLib:
    """Records the arguments of the pooled entries; last_hidden_pooled answers `rows` entries, row r the constant r + 10 * layer
    and token count r + 1, or ERR_INVALID when `cap` is too small for them."""

    def __init__(self, C_=4, rows=3):
        self.calls, self.C, self.rows = [], C_, rows

    def b200rwkv_last_error(self, h):
        return b"fake"

    def b200rwkv_keep_hidden_pooled(self, h, n, p, mode):
        layers = [] if n == 0 else np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int32)), (n,)).tolist()
        self.calls.append(("keep_hidden_pooled", n, layers, mode))
        return 0

    def b200rwkv_last_hidden_pooled(self, h, layer, p, cap, pn):
        self.calls.append(("last_hidden_pooled", layer, cap))
        if cap < self.rows * self.C:
            return capi.ERR_INVALID
        out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), (cap,))
        out[:self.rows * self.C] = np.repeat(np.arange(self.rows, dtype=np.float32) + 10 * layer, self.C)
        np.ctypeslib.as_array(C.cast(pn, C.POINTER(C.c_int32)), (self.rows,))[:] = np.arange(self.rows) + 1
        return self.rows


class _StubModel(runtime.Model):
    def __init__(self):
        self._h = None
        self.info = {"num_emb": 4, "num_vocab": 8}
        self.max_batch = 6
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


def test_keep_hidden_pooled_passes_layers_and_mode(fake):
    m = _StubModel()
    m.keep_hidden_pooled([5, 0, 2])
    m.keep_hidden_pooled([1], "mean")
    m.keep_hidden_pooled([1], capi.POOL_MEAN)
    m.keep_hidden_pooled([])
    assert fake.calls == [("keep_hidden_pooled", 3, [5, 0, 2], capi.POOL_LAST), ("keep_hidden_pooled", 1, [1], capi.POOL_MEAN),
                          ("keep_hidden_pooled", 1, [1], capi.POOL_MEAN), ("keep_hidden_pooled", 0, [], capi.POOL_LAST)]


def test_last_hidden_pooled_returns_rows_and_counts(fake):
    m = _StubModel()
    rows, ntok = m.last_hidden_pooled(2)
    assert fake.calls[-1] == ("last_hidden_pooled", 2, 6 * 4)              # room for max_batch entries by default
    assert rows.shape == (3, 4) and rows[:, 0].tolist() == [20, 21, 22] and ntok.tolist() == [1, 2, 3]
    with pytest.raises(capi.B200Error) as ei:
        m.last_hidden_pooled(2, max_rows=2)                                # small cap: the library's refusal comes through
    assert ei.value.code == capi.ERR_INVALID and fake.calls[-1] == ("last_hidden_pooled", 2, 2 * 4)


def test_embed_many_is_one_none_call_with_pooling_around_it(fake):
    m = _StubModel()
    e = m.embed_many([4, 1, 2], [[7, 8, 9], [3], [5, 6]], layer=1, mode="mean")
    assert m.infers == [([4, 1, 2], [3, 1, 2], [7, 8, 9, 3, 5, 6], [capi.OPTION_NONE] * 3)]
    assert fake.calls == [("keep_hidden_pooled", 1, [1], capi.POOL_MEAN), ("last_hidden_pooled", 1, 3 * 4),
                          ("keep_hidden_pooled", 0, [], capi.POOL_LAST)]
    assert e.shape == (3, 4) and e[:, 0].tolist() == [10, 11, 12]
    for slots, lists in (([0, 1], [[1]]), ([0, 1], [[1], []])):
        with pytest.raises(capi.B200Error):
            m.embed_many(slots, lists, layer=0)
