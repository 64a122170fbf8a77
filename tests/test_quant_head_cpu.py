"""CPU-side checks of the quantised vocabulary head (b200rwkv_head_format): the declaration and its ctypes binding against a C
compiler, the refusals made without an engine, runtime's format names, tests/head_oracle.quantize_head against each format's
quantize_model on a layer matrix of the same shape, and the head's bytes at the model shapes the project measures."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import quant_numpy as Q

import fp8_oracle as F8
import head_oracle as H
import int4_oracle as I4

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200rwkv.h")
FORMATS = {"Int8": capi.QUANT_INT8, "NF4": capi.QUANT_NF4, "FP8": capi.QUANT_FP8, "Int4": capi.QUANT_INT4}


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_binding_matches_the_header_as_compiled(tmp_path):
    assert "int32_t b200rwkv_head_format(b200rwkv_engine*, int32_t quant_type);" in open(HEADER).read()
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    assert sym["b200rwkv_head_format"] == (C.c_int32, [C.c_void_p, C.c_int32])
    assert capi.lib().b200rwkv_head_format.argtypes == [C.c_void_p, C.c_int32]
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    # the declaration has exactly the bound type, and the format values are the ones capi mirrors (compiled, not linked)
    checks = "".join(f'_Static_assert(B200RWKV_QUANT_{n} == {getattr(capi, "QUANT_" + n)}, "{n}");\n'
                     for n in ("NONE", "INT8", "NF4", "FP8", "INT4"))
    src = tmp_path / "decl.c"
    src.write_text('#include "b200rwkv.h"\n'
                   'int32_t (*const fn)(b200rwkv_engine*, int32_t) = b200rwkv_head_format;\n' + checks)
    subprocess.run([gcc, "-std=c11", "-Wall", "-Werror", "-c", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(tmp_path / "decl.o")], check=True)


def test_refusals_without_an_engine():
    L = capi.lib()
    assert L.b200rwkv_head_format(None, capi.QUANT_FP8) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    fake = C.c_void_p(16)          # never dereferenced: the value checks come first
    for bad in (-1, 7, 1 << 20):
        assert L.b200rwkv_head_format(fake, bad) == capi.ERR_INVALID
        assert "unknown quant_type" in _last_error()
    for unsupported in (3, 5):
        assert L.b200rwkv_head_format(fake, unsupported) == capi.ERR_UNSUPPORTED
        assert "SF4" in _last_error()


def test_runtime_format_names():
    for name, value in FORMATS.items():
        assert runtime.quant_kind(name) == value
        assert runtime.quant_kind(name.upper(), "quant_head") == value
    assert runtime.quant_kind("none") == capi.QUANT_NONE and runtime.quant_kind(capi.QUANT_FP8) == capi.QUANT_FP8
    for bad in ("fp16", "", "int 4"):
        with pytest.raises(capi.B200Error) as e:
            runtime.quant_kind(bad, "head_format")
        assert e.value.code == capi.ERR_INVALID and "head_format must be" in str(e.value)
    # the constructor checks its quant_head name before it creates anything
    with pytest.raises(capi.B200Error) as e:
        runtime.Model(synth.make_st("tiny6", 0), max_batch=1, quant_head="fp16")
    assert e.value.code == capi.ERR_INVALID and "quant_head must be" in str(e.value)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_quantize_head_is_the_layer_arithmetic(fmt):
    """quantize_head(w, q)["head.weight"] is what quantize_model makes of a layer matrix holding the same values; every other
    tensor is passed through untouched."""
    qt = FORMATS[fmt]
    rng = np.random.default_rng(qt)
    head = (rng.standard_normal((384, 256)) * 0.05).astype(np.float16)
    head[5] = 0
    head[9, 0] = np.float16(60000.0)
    other = (rng.standard_normal((256, 256)) * 0.05).astype(np.float16)
    w = {"head.weight": head, "blocks.0.att.key.weight": other, "emb.weight": head}
    got = H.quantize_head(w, qt)
    layer = H.QUANTIZE[qt]({"blocks.0.ffn.value.weight": head}, 1, qt)["blocks.0.ffn.value.weight"]
    assert got["head.weight"].dtype == layer.dtype and np.array_equal(got["head.weight"], layer)
    assert not np.array_equal(got["head.weight"].astype(np.float32), head.astype(np.float32))
    assert got["blocks.0.att.key.weight"] is other and got["emb.weight"] is head
    assert H.quantize_head(w, capi.QUANT_NONE)["head.weight"] is head
    # and it is the format's own dequantised matrix
    direct = {capi.QUANT_INT8: lambda m: Q.dequant_int8(*Q.quant_int8(m)), capi.QUANT_NF4: lambda m: Q.dequant_nf4(*Q.quant_nf4(m)),
              capi.QUANT_FP8: lambda m: F8.dequant_fp8(*F8.quant_fp8(m)), capi.QUANT_INT4: lambda m: I4.dequant_int4(*I4.quant_int4(m))}
    assert np.array_equal(got["head.weight"], direct[qt](head))


@pytest.mark.parametrize("preset,nbytes", [
    ("v6-7b", {"Int8": 276824064, "NF4": 142606336, "FP8": 268697600, "Int4": 142606336}),
    ("v6-3b", {"Int8": 173015040, "NF4": 89128960, "FP8": 168034304, "Int4": 89128960}),
    ("v7-2b9", {"Int8": 173015040, "NF4": 89128960, "FP8": 168034304, "Int4": 89128960}),
])
def test_head_bytes_at_the_measured_shapes(preset, nbytes):
    """The head's bytes per step in each format (quant_weight_bytes, which the engine's plans count), from the format
    definitions: codes of 8 or 4 bits plus f16 (min, max) / (scale, min) per 128 inputs, f16 absmax per 64, f32 per row."""
    s = synth.PRESETS[preset]
    V, Cm = s.V, s.C
    defs = {"Int8": V * Cm + V * (Cm // 128) * 4, "NF4": V * Cm // 2 + V * (Cm // 64) * 2, "FP8": V * Cm + V * 4,
            "Int4": V * Cm // 2 + V * (Cm // 128) * 4}
    for fmt, qt in FORMATS.items():
        b = H.head_bytes(V, Cm, qt)
        assert b == defs[fmt] == nbytes[fmt], fmt
        assert b < 2 * V * Cm
