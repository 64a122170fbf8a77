"""CPU-side checks of b200rwkv_infer_snapshots: the refusals it makes before it touches a device."""
import ctypes as C

import numpy as np

from ai00_server_b200 import capi


def test_null_engine_and_args_are_refused():
    slot, ntok, tok, opt = np.zeros(1, np.int32), np.ones(1, np.int32), np.zeros(1, np.uint32), np.zeros(1, np.int32)
    a = capi.InferArgs(C.sizeof(capi.InferArgs), 1, capi.ptr(slot).value, capi.ptr(ntok).value, capi.ptr(tok).value,
                       capi.ptr(opt).value, None, 0, None, None, None)
    entry, pos, ids = np.zeros(1, np.int32), np.ones(1, np.int32), np.zeros(1, np.uint64)
    lib = capi.lib()
    assert lib.b200rwkv_infer_snapshots(None, C.byref(a), 1, capi.ptr(entry), capi.ptr(pos), capi.ptr(ids)) == capi.ERR_INVALID
    assert lib.b200rwkv_infer_snapshots(None, None, 0, None, None, None) == capi.ERR_INVALID
    bad = capi.InferArgs(C.sizeof(capi.InferArgs) - 8, 1)
    assert lib.b200rwkv_infer_snapshots(None, C.byref(bad), 0, None, None, None) == capi.ERR_INVALID
    assert ids[0] == 0
