"""CPU-side checks of the in-place weight updates (b200rwkv_update_weights, b200rwkv_update_weights_device): the declarations
and their ctypes bindings, the b200rwkv_weight_src mirror against a C compiler, the refusals made without an engine, and that
the build has one weight-fill path (the recorded fills), which the updates replay."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from ai00_server_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200rwkv.h")
ENGINE = os.path.join(ROOT, "ai00_server_b200", "csrc", "engine.cu")


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def test_header_and_bindings_declare_the_entries():
    header = open(HEADER).read()
    assert "int32_t b200rwkv_update_weights(b200rwkv_engine*, const uint8_t* st, size_t len);" in header
    assert "int32_t b200rwkv_update_weights_device(b200rwkv_engine*, int32_t n, const b200rwkv_weight_src* src);" in header
    for name, value in (("F16", 0), ("BF16", 1), ("F32", 2)):
        assert re.search(rf"#define B200RWKV_DTYPE_{name}\s+{value}\b", header)
        assert getattr(capi, f"DTYPE_{name}") == value
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    P = C.c_void_p
    assert sym["b200rwkv_update_weights"] == (C.c_int32, [P, P, C.c_size_t])
    assert sym["b200rwkv_update_weights_device"] == (C.c_int32, [P, C.c_int32, C.POINTER(capi.WeightSrc)])
    for name in ("b200rwkv_update_weights", "b200rwkv_update_weights_device"):
        assert getattr(capi.lib(), name).argtypes == sym[name][1]


def test_weight_src_mirror_matches_the_header(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    exe = tmp_path / "layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200rwkv.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(b200rwkv_weight_src), offsetof(b200rwkv_weight_src, name),\n'
                   '  offsetof(b200rwkv_weight_src, dtype), offsetof(b200rwkv_weight_src, data)); return 0; }\n')
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    W = capi.WeightSrc
    assert got == [C.sizeof(W), W.name.offset, W.dtype.offset, W.data.offset]


def test_null_engine_image_and_table_are_refused():
    L = capi.lib()
    st = synth.make_st("tiny6", 0)
    assert L.b200rwkv_update_weights(None, capi.ptr(st), st.size) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    table = (capi.WeightSrc * 1)()
    table[0].name, table[0].dtype, table[0].data = b"head.weight", capi.DTYPE_F16, 16
    assert L.b200rwkv_update_weights_device(None, 1, table) == capi.ERR_INVALID
    assert "null engine" in _last_error()
    # a non-null handle that is never dereferenced: the image / table checks come first
    fake = C.c_void_p(16)
    assert L.b200rwkv_update_weights(fake, None, 64) == capi.ERR_INVALID
    assert "null image" in _last_error()
    assert L.b200rwkv_update_weights_device(fake, 1, None) == capi.ERR_INVALID
    assert "null tensor table" in _last_error()
    assert L.b200rwkv_update_weights_device(fake, 0, table) == capi.ERR_INVALID
    assert "n must be >= 1" in _last_error()
    table[0].data = None
    assert L.b200rwkv_update_weights_device(fake, 1, table) == capi.ERR_INVALID
    assert "null name or data" in _last_error()
    table[0].data, table[0].dtype = 16, 3
    assert L.b200rwkv_update_weights_device(fake, 1, table) == capi.ERR_INVALID
    assert "dtype" in _last_error()


def test_malformed_and_duplicate_images_are_refused_before_the_engine():
    L = capi.lib()
    fake = C.c_void_p(16)
    junk = (b"\xff" * 64)
    buf = (C.c_uint8 * len(junk)).from_buffer_copy(junk)
    assert L.b200rwkv_update_weights(fake, buf, len(junk)) == capi.ERR_INVALID
    assert "safetensors" in _last_error()
    # the same tensor named twice in one header
    hdr = b'{"a":{"dtype":"F16","shape":[1],"data_offsets":[0,2]},"a":{"dtype":"F16","shape":[1],"data_offsets":[0,2]}}'
    img = len(hdr).to_bytes(8, "little") + hdr + b"\x00\x00"
    buf = (C.c_uint8 * len(img)).from_buffer_copy(img)
    assert L.b200rwkv_update_weights(fake, buf, len(img)) == capi.ERR_INVALID
    assert "names a tensor twice" in _last_error()


def _body(src, signature):
    i = src.index(signature)
    return src[i:src.index("\n}\n", i)]


def test_weight_fills_have_one_path():
    """The build plans and records fills; only run_fill / fill_weights write weights.  Creation and both updates run those
    fills, so the layout an update writes is the one creation chose, decided once."""
    src = open(ENGINE).read()
    for sig in ("GemmLaunch b200rwkv_engine::make_launch(", "void b200rwkv_engine::build(const StFile& st) {",
                "float* b200rwkv_engine::vec_f32("):
        body = _body(src, sig)
        assert "<<<" not in body and "cudaMemcpy" not in body, sig
    run_fill = _body(src, "void b200rwkv_engine::run_fill(")
    fill_weights = _body(src, "void b200rwkv_engine::fill_weights(")
    for kern in ("quantize_fp8_kernel<<<", "quantize_int4_kernel<<<", "quantize_weight_kernel<QT_INT8><<<",
                 "quantize_weight_kernel<QT_NF4><<<", "launch_f16_to_f32(", "launch_decay_table(", "wd2_k_major("):
        assert kern in run_fill, kern
    assert "run_fill(" in fill_weights and "to_f16_kernel" in fill_weights
    # creation and both updates go through fill_weights
    assert "fill_weights(in);" in _body(src, "void b200rwkv_engine::build(const StFile& st) {")
    assert "fill_weights(in);" in _body(src, "int32_t b200rwkv_update_weights(")
    assert "fill_weights(in);" in _body(src, "int32_t b200rwkv_update_weights_device(")
