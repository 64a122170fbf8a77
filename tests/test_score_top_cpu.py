"""CPU-side checks of top-n log-probabilities (b200rwkv_score_top / b200rwkv_last_score_top): the ctypes bindings against the
header, the refusals the two entries make before touching a device, and the bookkeeping of Model.score_top,
Model.last_score_top, infer_ex(top_n=...) and perplexity(top_n=...) with the library stubbed out."""
import ctypes as C
import pathlib
import re

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime

HEADER = pathlib.Path(__file__).resolve().parent.parent / "include" / "b200rwkv.h"


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_bindings_match_the_header():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert sym["b200rwkv_score_top"] == (C.c_int32, [C.c_void_p, C.c_int32])
    assert sym["b200rwkv_last_score_top"] == (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t])
    text = HEADER.read_text()
    assert re.search(r"int32_t b200rwkv_score_top\(b200rwkv_engine\*, int32_t top_n\);", text)
    assert re.search(r"int32_t b200rwkv_last_score_top\(b200rwkv_engine\*, uint32_t\* ids_out, float\* logprobs_out, "
                     r"size_t cap\);", text)
    L = capi.lib()
    assert L.b200rwkv_score_top.argtypes == sym["b200rwkv_score_top"][1]
    assert L.b200rwkv_last_score_top.argtypes == sym["b200rwkv_last_score_top"][1]


def test_score_top_refusals_without_an_engine():
    """n outside [0, 128] is ERR_INVALID before anything else; a valid n still needs an engine."""
    L = capi.lib()
    for n in (-1, 129, 1000, -(2 ** 31)):
        assert L.b200rwkv_score_top(None, n) == capi.ERR_INVALID
        assert "top_n must be in [0, 128]" in _last_error()
    for n in (0, 1, 128):
        assert L.b200rwkv_score_top(None, n) == capi.ERR_INVALID
        assert "null engine" in _last_error()


def test_last_score_top_refuses_a_null_engine():
    L = capi.lib()
    buf = np.zeros(8, np.uint32)
    assert L.b200rwkv_last_score_top(None, capi.ptr(buf), capi.ptr(buf), buf.size) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    assert L.b200rwkv_last_score_top(None, None, None, 0) == capi.ERR_INVALID


class _FakeLib:
    """score_top records its setting; infer_ex scores every SCORE token (score = -token, argmax = token); last_score_top
    answers rows [r][k] = 100 r + k for the last call's scored tokens, or ERR_STATE if it ran with the setting off."""

    def __init__(self):
        self.calls, self.n, self.last = [], 0, None

    def b200rwkv_last_error(self, h):
        return b"fake"

    def b200rwkv_score_top(self, h, n):
        self.calls.append(("score_top", n))
        self.n = n
        return 0

    def b200rwkv_infer_ex(self, h, args):
        a = args._obj
        n = a.nslot
        ntok = np.ctypeslib.as_array(C.cast(a.ntok, C.POINTER(C.c_int32)), (n,))
        opt = np.ctypeslib.as_array(C.cast(a.option, C.POINTER(C.c_int32)), (n,))
        toks = np.ctypeslib.as_array(C.cast(a.tokens, C.POINTER(C.c_uint32)), (int(ntok.sum()),))
        sc = [t for i in range(n) if opt[i] == capi.OPTION_SCORE for t in toks[ntok[:i].sum():ntok[:i + 1].sum()]]
        if sc:
            np.ctypeslib.as_array(C.cast(a.score_out, C.POINTER(C.c_float)), (len(sc),))[:] = -np.asarray(sc, np.float32)
            np.ctypeslib.as_array(C.cast(a.argmax_out, C.POINTER(C.c_uint32)), (len(sc),))[:] = sc
        self.calls.append(("infer_ex", ntok.tolist(), opt.tolist()))
        self.last = (self.n, len(sc))
        return 0

    def b200rwkv_last_score_top(self, h, ids, lp, cap):
        self.calls.append(("last_score_top", cap))
        n, rows = self.last
        if n == 0:
            return capi.ERR_STATE
        if ids is None and lp is None:
            return rows
        if cap < rows * n:
            return capi.ERR_INVALID
        v = (100 * np.arange(rows)[:, None] + np.arange(n)[None, :]).ravel()
        np.ctypeslib.as_array(C.cast(ids, C.POINTER(C.c_uint32)), (rows * n,))[:] = v
        np.ctypeslib.as_array(C.cast(lp, C.POINTER(C.c_float)), (rows * n,))[:] = -v
        return rows


class _StubModel(runtime.Model):
    def __init__(self):
        self._h = None
        self._top_n = 0
        self.info = {"num_emb": 4, "num_vocab": 8}
        self.max_batch = 6


@pytest.fixture
def fake():
    real, f = capi._lib, _FakeLib()
    capi._lib = f
    yield f
    capi._lib = real


def test_infer_ex_top_n_sets_runs_reads_and_restores(fake):
    m = _StubModel()
    m.score_top(3)
    rows, scores, tops = m.infer_ex([0, 1, 2], [2, 1, 3], [5, 6, 7, 1, 2, 3],
                                    [capi.OPTION_SCORE, capi.OPTION_LAST, capi.OPTION_SCORE], top_n=4)
    assert [c[0] for c in fake.calls] == ["score_top", "score_top", "infer_ex", "last_score_top", "last_score_top",
                                          "score_top"]
    assert fake.calls[1] == ("score_top", 4) and fake.calls[-1] == ("score_top", 3) and m._top_n == 3
    assert tops[1] is None and scores[1] is None
    assert tops[0][0].shape == (2, 4) and tops[2][0].shape == (3, 4)
    assert tops[0][0][1].tolist() == [100, 101, 102, 103] and tops[2][0][0].tolist() == [200, 201, 202, 203]
    assert tops[2][1][2].tolist() == [-400, -401, -402, -403]
    assert scores[2][1].tolist() == [1, 2, 3]
    assert len(m.infer_ex([0], [1], [5], [capi.OPTION_SCORE])) == 2        # without top_n: (rows, scores) as before


def test_last_score_top_with_the_setting_off_raises(fake):
    m = _StubModel()
    m.infer_ex([0], [1], [5], [capi.OPTION_SCORE])
    with pytest.raises(capi.B200Error) as ei:
        m.last_score_top()
    assert ei.value.code == capi.ERR_STATE


def test_perplexity_top_n_aligns_lists_with_the_tokens(fake):
    m = _StubModel()
    p0 = m.perplexity(0, [4, 5, 6])
    p1, (ids, lp) = m.perplexity(0, [4, 5, 6], top_n=2)
    assert p0 == p1
    assert ids.tolist() == [[100, 101], [200, 201], [300, 301]]             # token 0 fed first: its row is dropped
    ph, (ids, _) = m.perplexity(0, [4, 5, 6], head=0.5, top_n=2)
    assert ph == m.perplexity(0, [4, 5, 6], head=0.5)
    assert ids.tolist() == [[0, 1], [100, 101], [200, 201]]                 # with head: token 0's list is the kept row's
    assert m._top_n == 0
