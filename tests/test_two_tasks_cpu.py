"""The error text of the C ABI is per thread (include/b200rwkv.h: "the infer task and the softmax task never see each other's
text"), checked on the host-only entries, so no GPU is needed.  Two threads fail at once -- one in b200rwkv_info_from_st
on a malformed image, the other in b200rwkv_read_state with a bad b200rwkv_info -- and a barrier makes both failures land
before either thread reads b200rwkv_last_error.  Each must read its own message, and read it unchanged after the other
thread's successful host-only call.  A process-wide error string fails this: one thread would read the other's text.
tests/test_gpu_two_tasks.py checks the same on an engine's infer and sampling entries."""
import ctypes as C
import dataclasses
import threading

import numpy as np

from ai00_server_b200 import capi, synth

ROUNDS = 8
TIMEOUT = 60.0


def last_error():
    msg = capi.lib().b200rwkv_last_error(None)
    return msg.decode("utf-8", "replace") if msg else ""


def test_error_text_is_per_thread():
    lib = capi.lib()
    good = synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], time_state=True), 0)
    good_info = capi.Info(**capi.info_from_st(good))
    junk = np.frombuffer(b"\x10\x00\x00\x00\x00\x00\x00\x00{\"a\":1}        ", dtype=np.uint8).copy()
    bad_info = capi.Info(**{**good_info.as_dict(), "num_emb": good_info.num_emb + 64})       # num_emb != num_head * head_size
    out = np.empty((good_info.num_layer, good_info.head_size + 2, good_info.num_emb), np.float32)
    bar = threading.Barrier(2, timeout=TIMEOUT)
    seen = {"st": [], "state": []}
    errors = []

    def st_thread():
        for _ in range(ROUNDS):
            info = capi.Info()
            bar.wait()
            code = lib.b200rwkv_info_from_st(capi.ptr(junk), junk.size, C.byref(info))
            bar.wait()                                  # both calls have failed
            first = last_error()
            bar.wait()
            ok = lib.b200rwkv_info_from_st(capi.ptr(good), good.size, C.byref(info))
            bar.wait()                                  # both successful calls have returned
            seen["st"].append((code, first, ok, last_error()))

    def state_thread():
        state = np.empty_like(out)
        for _ in range(ROUNDS):
            bar.wait()
            code = lib.b200rwkv_read_state(C.byref(bad_info), capi.ptr(good), good.size, capi.ptr(state))
            bar.wait()
            first = last_error()
            bar.wait()
            ok = lib.b200rwkv_read_state(C.byref(good_info), capi.ptr(good), good.size, capi.ptr(state))
            bar.wait()
            seen["state"].append((code, first, ok, last_error()))

    def run(body):
        def wrapped():
            try:
                body()
            except BaseException as ex:                 # noqa: BLE001 -- reported below
                errors.append(ex)
                bar.abort()
        return wrapped

    threads = [threading.Thread(target=run(b), daemon=True) for b in (st_thread, state_thread)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(TIMEOUT)
    assert not any(t.is_alive() for t in threads), "a thread did not finish"
    assert not errors, errors
    assert len(seen["st"]) == len(seen["state"]) == ROUNDS
    for code, first, ok, again in seen["st"]:
        assert code == capi.ERR_INVALID and ok == capi.OK
        assert first and "bad model info" not in first, first
        assert again == first
    for code, first, ok, again in seen["state"]:
        assert code == capi.ERR_INVALID and ok == capi.OK
        assert first == "bad model info", first
        assert again == first
    assert len({f for _, f, _, _ in seen["st"]}) == 1            # the same failure gives the same text every round

