"""CPU-side checks of adapters on quantised layers (b200rwkv_options.quant_adapters): the header layout against the ctypes
mirror, the previous options size, every refusal before any CUDA call, the host checks the flag relaxes (and the ones it
keeps), and the flag's way through runtime.Model."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

QUANTS = (capi.QUANT_INT8, capi.QUANT_NF4, capi.QUANT_FP8, capi.QUANT_INT4)


def _last_error():
    return capi.lib().b200rwkv_last_error(None).decode()


def _opt(**kw):
    opt = capi.Options()
    opt.struct_bytes = C.sizeof(capi.Options)
    opt.max_batch, opt.token_chunk_size = 2, 32
    for k, v in kw.items():
        setattr(opt, k, v)
    return opt


def _adapters(st, files, opt):
    h = C.c_void_p()
    n = len(files)
    ptrs = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_size_t * n)(*[f.size for f in files])
    alphas = (C.c_float * n)(*([1.0] * n))
    rc = capi.lib().b200rwkv_create_adapters(capi.ptr(st), st.size, C.byref(opt), n, C.cast(ptrs, C.c_void_p),
                                             C.cast(lens, C.c_void_p), C.cast(alphas, C.c_void_p), C.byref(h))
    if h:               # a call that passed every check on a machine with a GPU built an engine
        capi.lib().b200rwkv_destroy(h)
    return rc


def _places(st, n, targets, opt):
    h = C.c_void_p()
    rc = capi.lib().b200rwkv_create_adapter_places(capi.ptr(st), st.size, C.byref(opt), n, targets, C.byref(h))
    if h:
        capi.lib().b200rwkv_destroy(h)
    return rc


def _past_host_checks(rc):
    """Without a GPU a call that passed every host check ends at the device check; with one it builds."""
    assert rc in (capi.OK, capi.ERR_CUDA), _last_error()
    if rc == capi.ERR_CUDA:
        assert "no CPU fallback" in _last_error()


@pytest.fixture(scope="module")
def tiny6():
    return synth.make_st("tiny6", 0)


def test_header_layout_matches_the_ctypes_mirror(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200rwkv.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(b200rwkv_options), offsetof(b200rwkv_options, quant_adapters),\n'
                   '  offsetof(b200rwkv_options, batch_invariant)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    # the field fills the tail padding: the struct keeps its size
    assert got == [152, 148, 144]
    assert [C.sizeof(capi.Options), capi.Options.quant_adapters.offset, capi.Options.batch_invariant.offset] == got


def test_bindings_declare_the_operator_entry():
    sym = {name: (res, args) for name, res, args in capi.SYMBOLS}
    P = C.c_void_p
    assert sym["b200rwkv_op_gemm_tail"] == (C.c_int32, [C.c_int32] * 5 + [C.POINTER(capi.GemmSeg), P, P, C.POINTER(C.c_int32 * 4)])


def test_refusals_come_before_any_cuda_call(tiny6):
    h = C.c_void_p()
    L = capi.lib()
    ad = synth.make_lora_st("tiny6", rank=4, seed=1)
    for v in (2, -1):
        opt = _opt(quant_adapters=v, quant_layers=6, quant_type=capi.QUANT_INT8)
        assert L.b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(opt), C.byref(h)) == capi.ERR_INVALID
        assert "quant_adapters" in _last_error()
        assert _adapters(tiny6, [ad], opt) == capi.ERR_INVALID
        assert "quant_adapters" in _last_error()
        assert _places(tiny6, 1, capi.TARGET_ATT_K, opt) == capi.ERR_INVALID
        assert "quant_adapters" in _last_error()
    two = _opt(quant_adapters=1, num_devices=2)
    two.devices[0], two.devices[1] = 0, 1
    assert L.b200rwkv_create_ex(capi.ptr(tiny6), tiny6.size, C.byref(two), C.byref(h)) == capi.ERR_UNSUPPORTED
    assert "one GPU" in _last_error()
    assert _adapters(tiny6, [ad], two) == capi.ERR_UNSUPPORTED
    assert _places(tiny6, 1, capi.TARGET_ATT_K, two) == capi.ERR_UNSUPPORTED
    assert not h.value
    # the operator entry checks its tail count first
    seg = capi.GemmSeg(128, 128, None, None, None, 0, 0, 0, None, None, None, 128, None)
    e = np.zeros((128, 128), np.float16)
    for n in (0, 9):
        assert L.b200rwkv_op_gemm_tail(0, 1, capi.QUANT_INT8, 0, n, C.byref(seg), capi.ptr(e), capi.ptr(e), None) == capi.ERR_INVALID


def test_previous_options_size_reads_the_flag_as_off(tiny6):
    """struct_bytes = offsetof(batch_invariant): the field is not read, so a pair on a quantised layer stays refused."""
    ad = synth.make_lora_st("tiny6", rank=4, seed=1)
    old = _opt(quant_adapters=1, quant_layers=6, quant_type=capi.QUANT_INT8)
    old.struct_bytes = capi.Options.batch_invariant.offset
    assert _adapters(tiny6, [ad], old) == capi.ERR_UNSUPPORTED
    assert "quantised" in _last_error()
    assert _places(tiny6, 1, capi.TARGET_ATT_K | capi.TARGET_FFN_V, old) == capi.ERR_UNSUPPORTED
    assert "name no f16 projection matrix" in _last_error()


@pytest.mark.parametrize("qt", QUANTS)
def test_the_flag_lets_adapters_reach_quantised_layers(tiny6, qt):
    ad = synth.make_lora_st("tiny6", rank=8, seed=1)
    off = _opt(quant_layers=6, quant_type=qt)
    assert _adapters(tiny6, [ad], off) == capi.ERR_UNSUPPORTED
    assert "quantised" in _last_error()
    on = _opt(quant_layers=6, quant_type=qt, quant_adapters=1)
    _past_host_checks(_adapters(tiny6, [ad, synth.make_lora_st("tiny6", rank=128, seed=2)], on))
    # places: every layer quantised, so without the flag only the head could be targeted
    targets = capi.TARGET_ATT_K | capi.TARGET_FFN_V
    assert _places(tiny6, 2, targets, off) == capi.ERR_UNSUPPORTED
    _past_host_checks(_places(tiny6, 2, targets, on))


def test_the_flag_keeps_the_other_file_checks(tiny6):
    on = _opt(quant_layers=6, quant_type=capi.QUANT_INT4, quant_adapters=1)
    C_, F = 256, 896
    pairs = lambda **t: synth.pack_st({k: np.asarray(v, np.float16) for k, v in t.items()})
    r129 = pairs(**{"blocks.0.ffn.value.lora.0": np.zeros((F, 129)), "blocks.0.ffn.value.lora.1": np.zeros((C_, 129))})
    assert _adapters(tiny6, [r129], on) == capi.ERR_UNSUPPORTED
    assert "above 128" in _last_error()
    full = synth.pack_st({"blocks.0.att.key.weight": np.zeros((C_, C_), np.float16)})
    assert _adapters(tiny6, [full], on) == capi.ERR_UNSUPPORTED
    assert "full tensor" in _last_error()
    bad = pairs(**{"blocks.0.att.key.lora.0": np.zeros((C_ + 8, 4)), "blocks.0.att.key.lora.1": np.zeros((C_, 4))})
    assert _adapters(tiny6, [bad], on) == capi.ERR_INVALID
    assert "shapes" in _last_error()


def test_model_passes_the_flag_through(tiny6):
    seen = []

    class FakeLib:
        def b200rwkv_create_ex(self, st, n, opt, h):
            o = opt._obj
            seen.append((o.struct_bytes, o.quant_adapters, o.quant_layers, o.quant_type))
            return capi.ERR_UNSUPPORTED

        def b200rwkv_last_error(self, engine):
            return b"stub"

    real = capi._lib
    capi._lib = FakeLib()
    try:
        for flag in (True, False):
            with pytest.raises(capi.B200Error):
                runtime.Model(tiny6, max_batch=3, quant=2, quant_type="Int4", quant_adapters=flag, devices=[0])
    finally:
        capi._lib = real
    assert seen == [(C.sizeof(capi.Options), 1, 2, capi.QUANT_INT4), (C.sizeof(capi.Options), 0, 2, capi.QUANT_INT4)]
