"""CPU-side checks of the whole-distribution sampling entry (b200rwkv_sample_probs): its ctypes binding, the refusals it makes
before touching a device, and the argument packing of Model.sample_probs with the library stubbed out."""
import ctypes as C

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_binding_declares_the_entry():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert sym["b200rwkv_sample_probs"] == (C.c_int32, [C.c_void_p, C.c_int32] + [C.c_void_p] * 9)
    assert capi.lib().b200rwkv_sample_probs.argtypes == sym["b200rwkv_sample_probs"][1]


def test_refusals_without_an_engine():
    """nrows < 1, NULL slots or output, offsets that descend or go negative, and entries without token / value arrays are
    ERR_INVALID before any CUDA call; well-formed arguments reach the engine check."""
    L = capi.lib()
    slots = np.array([0, 1], np.int32)
    out = np.zeros((2, 8), np.float32)
    tok = np.array([1, 2, 3], np.uint32)
    val = np.array([0.5, 0.25, 1.0], np.float32)
    P = capi.ptr

    def call(nrows=2, sl=P(slots), po=None, pt=P(tok), pv=P(val), bo=None, bt=P(tok), bv=P(val), o=P(out)):
        keep = [np.asarray(x, np.int32) if x is not None else None for x in (po, bo)]
        a = [P(k) if k is not None else None for k in keep]
        return L.b200rwkv_sample_probs(None, nrows, sl, a[0], pt, pv, None, a[1], bt, bv, o)

    cases = {
        "nrows = 0": (lambda: call(nrows=0), "bad argument"),
        "nrows < 0": (lambda: call(nrows=-3), "bad argument"),
        "null slots": (lambda: call(sl=None), "bad argument"),
        "null output": (lambda: call(o=None), "bad argument"),
        "descending penalty offsets": (lambda: call(po=[0, 2, 1]), "penalty offsets must ascend"),
        "negative penalty offset": (lambda: call(po=[-1, 0, 1]), "penalty offsets must ascend"),
        "descending bias offsets": (lambda: call(bo=[1, 0, 2]), "bias offsets must ascend"),
        "penalties without tokens": (lambda: call(po=[0, 1, 3], pt=None), "bad adjustment lists"),
        "bias without values": (lambda: call(bo=[0, 0, 1], bv=None), "bad adjustment lists"),
        "negative list length": (lambda: call(po=[0, 0, -2]), "bad adjustment lists"),
    }
    for name, (fn, text) in cases.items():
        assert fn() == capi.ERR_INVALID, name
        assert text in _last_error(), (name, _last_error())
    for ok in (lambda: call(), lambda: call(po=[0, 1, 3], bo=[0, 0, 2]), lambda: call(nrows=1, po=[0, 0], pt=None, pv=None)):
        assert ok() == capi.ERR_INVALID and "null engine" in _last_error()


class _FakeLib:
    """Records what b200rwkv_sample_probs receives and fills row i with the constant i."""

    def __init__(self, V):
        self.V, self.seen = V, None

    def b200rwkv_sample_probs(self, h, n, sl, po, pt, pv, bits, bo, bt, bv, out):
        arr = lambda p, t, k: np.ctypeslib.as_array(C.cast(p, C.POINTER(t)), (k,)).copy()
        po_, bo_ = arr(po, C.c_int32, n + 1), arr(bo, C.c_int32, n + 1)
        words = (self.V + 31) // 32
        self.seen = dict(slots=arr(sl, C.c_int32, n).tolist(), po=po_.tolist(), bo=bo_.tolist(),
                         pt=arr(pt, C.c_uint32, po_[-1]).tolist() if po_[-1] else [], pv=arr(pv, C.c_float, po_[-1]).tolist() if po_[-1] else [],
                         bt=arr(bt, C.c_uint32, bo_[-1]).tolist() if bo_[-1] else [], bv=arr(bv, C.c_float, bo_[-1]).tolist() if bo_[-1] else [],
                         bits=None if bits is None else arr(bits, C.c_uint32, n * words).reshape(n, words))
        o = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_float)), (n, self.V))
        o[:] = np.arange(n, dtype=np.float32)[:, None]
        return 0


class _StubModel(runtime.Model):
    def __init__(self, V):
        self._h = None
        self.info = {"num_vocab": V}


@pytest.fixture
def fake():
    real, f = capi._lib, _FakeLib(40)
    capi._lib = f
    yield f
    capi._lib = real


def test_sample_probs_packs_the_lists_as_sample_topk_does(fake):
    m = _StubModel(40)
    allow = np.ones((2, 40), bool)
    allow[1, [0, 33, 39]] = False
    got = m.sample_probs([3, 1], penalties=[{7: 0.5, 2: 1.5}, None], bias=[None, {39: -1.0}], allow=allow)
    assert got.shape == (2, 40) and got.dtype == np.float32 and (got[1] == 1).all()
    s = fake.seen
    assert s["slots"] == [3, 1] and s["po"] == [0, 2, 2] and s["pt"] == [7, 2] and s["pv"] == [0.5, 1.5]
    assert s["bo"] == [0, 0, 1] and s["bt"] == [39] and s["bv"] == [-1.0]
    assert s["bits"].shape == (2, 2)
    unpacked = np.unpackbits(s["bits"].view(np.uint8), bitorder="little").reshape(2, 64)[:, :40].astype(bool)
    assert np.array_equal(unpacked, allow)
    m.sample_probs([0])
    assert fake.seen["bits"] is None and fake.seen["po"] == [0, 0] and fake.seen["bo"] == [0, 0]
