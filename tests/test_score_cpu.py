"""CPU-side checks of the scoring entry (b200rwkv_infer_ex with B200RWKV_OPTION_SCORE): the ctypes mirror of its argument
struct, the refusals it makes before touching a device, and the bookkeeping of Model.perplexity (the reference's
perplexity(), run.rs:699-755) with the engine stubbed out."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_infer_args_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "sz.c"
    fields = [n for n, _ in capi.InferArgs._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200rwkv.h"\n'
                   'int main(void) { printf("%zu %d\\n", sizeof(b200rwkv_infer_args), B200RWKV_OPTION_SCORE);\n'
                   + "".join(f'  printf("%zu\\n", offsetof(b200rwkv_infer_args, {f}));\n' for f in fields)
                   + "  return 0; }\n")
    exe = tmp_path / "sz"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[:2] == [C.sizeof(capi.InferArgs), capi.OPTION_SCORE]
    assert got[2:] == [getattr(capi.InferArgs, f).offset for f in fields]


def _args(**kw):
    slot, ntok, tok, opt = (np.zeros(1, np.int32), np.ones(1, np.int32), np.zeros(1, np.uint32),
                            np.full(1, capi.OPTION_SCORE, np.int32))
    score = np.zeros(1, np.float32)
    a = capi.InferArgs(C.sizeof(capi.InferArgs), 1, capi.ptr(slot).value, capi.ptr(ntok).value, capi.ptr(tok).value,
                       capi.ptr(opt).value, None, 0, None, capi.ptr(score).value, None)
    for k, v in kw.items():
        setattr(a, k, v)
    return a, (slot, ntok, tok, opt, score)


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_infer_ex_refusals_without_an_engine():
    """Refused before any CUDA call: a NULL argument struct, a struct_bytes that is not sizeof(b200rwkv_infer_args) (an
    older or newer caller), and a NULL engine."""
    L = capi.lib()
    assert L.b200rwkv_infer_ex(None, None) == capi.ERR_INVALID
    assert "null args" in _last_error()
    for wrong in (0, C.sizeof(capi.InferArgs) - 8, C.sizeof(capi.InferArgs) + 8):
        a, keep = _args(struct_bytes=wrong)
        assert L.b200rwkv_infer_ex(None, C.byref(a)) == capi.ERR_INVALID
        assert "struct_bytes" in _last_error()
    a, keep = _args()
    assert L.b200rwkv_infer_ex(None, C.byref(a)) == capi.ERR_INVALID
    assert "null engine" in _last_error()


class _StubModel(runtime.Model):
    """Model.perplexity over a fake infer_ex: the score of fed token j is -(j + 1) / 8 (exact in f32), NaN for token 0."""

    def __init__(self):
        self.calls = []
        self._h = None

    def infer_ex(self, slots, ntok, tokens, options):
        self.calls.append((list(slots), list(ntok), list(tokens), list(options)))
        s = -(np.arange(ntok[0], dtype=np.float32) + 1) / 8
        s[0] = np.nan
        return [np.zeros((0, 4), np.float32)], [(s, np.zeros(ntok[0], np.uint32))]


def test_perplexity_bookkeeping():
    m = _StubModel()
    toks = [7, 3, 9, 11]
    # no head: a token 0 goes first, scores of fed tokens 1..4 are used, the divisor is len + 1
    got = m.perplexity(2, toks)
    assert m.calls[-1] == ([2], [5], [0] + toks, [capi.OPTION_SCORE])
    assert got == pytest.approx((2 + 3 + 4 + 5) / 8 / 5, rel=1e-7)
    # head: ln(head) replaces the first score, the kept row's score of tokens[0] is not used, the divisor is len
    got = m.perplexity(1, toks, head=0.25)
    assert m.calls[-1] == ([1], [4], toks, [capi.OPTION_SCORE])
    assert got == pytest.approx(-(np.log(0.25) - (2 + 3 + 4) / 8) / 4, rel=1e-6)
    # one token with a head: only ln(head)
    assert m.perplexity(0, [5], head=0.5) == pytest.approx(-np.log(0.5), rel=1e-6)
    assert np.isfinite(m.perplexity(0, [5]))           # [0, 5]: one used score over two tokens


def test_infer_ex_splits_scores_by_entry_order():
    """Model.infer_ex hands each SCORE entry its own slice of score_out / argmax_out, in entry order, whatever sits between."""
    calls = {}

    class FakeLib:
        def b200rwkv_infer_ex(self, h, ref):
            a = ref._obj
            n = a.nslot
            ntok = np.ctypeslib.as_array(C.cast(a.ntok, C.POINTER(C.c_int32)), (n,))
            opt = np.ctypeslib.as_array(C.cast(a.option, C.POINTER(C.c_int32)), (n,))
            nscore = int(sum(t for t, o in zip(ntok, opt) if o == capi.OPTION_SCORE))
            score = np.ctypeslib.as_array(C.cast(a.score_out, C.POINTER(C.c_float)), (nscore,))
            amax = np.ctypeslib.as_array(C.cast(a.argmax_out, C.POINTER(C.c_uint32)), (nscore,))
            rows = np.ctypeslib.as_array(C.cast(a.rows_out, C.POINTER(C.c_int32)), (n,))
            score[:] = np.arange(nscore)
            amax[:] = np.arange(nscore) + 100
            rows[:] = [t if o == capi.OPTION_FULL else (1 if o == capi.OPTION_LAST and t else 0) for t, o in zip(ntok, opt)]
            calls["struct_bytes"] = a.struct_bytes
            return 0

    m = _StubModel()
    m.info = {"num_vocab": 4}
    real = capi._lib
    capi._lib = FakeLib()
    try:
        rows, scores = runtime.Model.infer_ex(m, [3, 0, 1, 2], [2, 3, 1, 4],
                                              list(range(8)), [capi.OPTION_SCORE, capi.OPTION_FULL, capi.OPTION_LAST, capi.OPTION_SCORE])
    finally:
        capi._lib = real
    assert calls["struct_bytes"] == C.sizeof(capi.InferArgs)
    assert [r.shape[0] for r in rows] == [0, 3, 1, 0]
    assert scores[1] is None and scores[2] is None
    assert scores[0][0].tolist() == [0, 1] and scores[0][1].tolist() == [100, 101]
    assert scores[3][0].tolist() == [2, 3, 4, 5] and scores[3][1].tolist() == [102, 103, 104, 105]
