"""CPU-side checks of the batch-invariant option (b200rwkv_options.batch_invariant, b200rwkv_ln_args.batch_invariant): the
header layout against the ctypes mirrors, the previous options size, every refusal before any CUDA call, and the flag's
way through runtime.Model."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from ai00_server_b200 import capi, runtime, synth


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def _opt(**kw):
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    for k, v in kw.items():
        setattr(opt, k, v)
    return opt


@pytest.fixture(scope="module")
def tiny6():
    return synth.make_st("tiny6", 0)


def test_header_layout_matches_the_ctypes_mirrors(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200rwkv.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(b200rwkv_options), offsetof(b200rwkv_options, batch_invariant),\n'
                   '  sizeof(b200rwkv_ln_args), offsetof(b200rwkv_ln_args, batch_invariant)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(capi.Options), capi.Options.batch_invariant.offset, C.sizeof(capi.LnArgs),
                   capi.LnArgs.batch_invariant.offset]
    # the field is the last one of both structs: the options size before it is its offset
    assert capi.Options.batch_invariant.offset == capi.Options.quant_type.offset + 4


def test_previous_options_size_passes_the_host_checks_and_reads_as_off(tiny6):
    """struct_bytes = offsetof(batch_invariant) is accepted and the field is not read: a bad device count behind it is
    the error, not the size or the (unread) flag."""
    h = C.c_void_p()
    opt = _opt(num_devices=3, batch_invariant=7)
    opt.struct_bytes = capi.Options.batch_invariant.offset
    assert capi.lib().b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(opt), C.byref(h)) == capi.ERR_INVALID
    assert "num_devices" in _last_error()
    bad = _opt()
    bad.struct_bytes = capi.Options.batch_invariant.offset - 4
    assert capi.lib().b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(bad), C.byref(h)) == capi.ERR_INVALID
    assert "struct_bytes" in _last_error()
    # the adapters constructors accept the previous size too: their own checks come next
    old = _opt()
    old.struct_bytes = capi.Options.batch_invariant.offset
    assert capi.lib().b200rwkv_create_adapter_places(capi.ptr(tiny6), tiny6.size, C.byref(old), 0, 1, C.byref(h)) == capi.ERR_INVALID
    assert "adapter places" in _last_error()


def test_refusals_come_before_any_cuda_call(tiny6):
    h = C.c_void_p()
    L = capi.lib()
    for v in (2, -1, 255):
        assert L.b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(_opt(batch_invariant=v)), C.byref(h)) == capi.ERR_INVALID
        assert "batch_invariant" in _last_error()
    opt = _opt(batch_invariant=1, num_devices=2)
    opt.devices[0], opt.devices[1] = 0, 1
    assert L.b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(opt), C.byref(h)) == capi.ERR_UNSUPPORTED
    assert "batch-invariant" in _last_error()
    ad = synth.make_lora_st("tiny6", rank=4, seed=1)
    ptrs, lens, alphas = (C.c_void_p * 1)(ad.ctypes.data), (C.c_size_t * 1)(ad.size), (C.c_float * 1)(1.0)
    assert L.b200rwkv_create_adapters(capi.ptr(tiny6), tiny6.size, C.byref(_opt(batch_invariant=1)), 1, C.cast(ptrs, C.c_void_p),
                                      C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p), C.byref(h)) == capi.ERR_UNSUPPORTED
    assert "batch-invariant" in _last_error()
    assert L.b200rwkv_create_adapter_places(capi.ptr(tiny6), tiny6.size, C.byref(_opt(batch_invariant=1)), 2,
                                            capi.TARGET_ATT_K, C.byref(h)) == capi.ERR_UNSUPPORTED
    assert "batch-invariant" in _last_error()
    assert not h.value
    # op_ln: a flag other than 0 / 1 is refused before the step is built
    a = capi.LnArgs(stage=capi.LN_MIX, C=256, S=1, nslot=0, launches=1, batch_invariant=2)
    assert L.b200rwkv_op_ln(0, C.byref(a)) == capi.ERR_INVALID
    assert "batch_invariant" in _last_error()


def test_model_passes_the_flag_through(tiny6):
    seen = []

    class FakeLib:
        def b200rwkv_create_ex(self, st, n, opt, h):
            o = opt._obj
            seen.append((o.struct_bytes, o.batch_invariant, o.max_batch, o.token_chunk_size))
            return capi.ERR_UNSUPPORTED

        def b200rwkv_last_error(self, engine):
            return b"stub"

    real = capi._lib
    capi._lib = FakeLib()
    try:
        for flag in (True, False):
            with pytest.raises(capi.B200Error):
                runtime.Model(tiny6, max_batch=3, token_chunk_size=64, batch_invariant=flag, devices=[0])
    finally:
        capi._lib = real
    assert seen == [(C.sizeof(capi.Options), 1, 3, 64), (C.sizeof(capi.Options), 0, 3, 64)]
