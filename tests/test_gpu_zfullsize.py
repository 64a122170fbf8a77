"""BASELINE.json's shapes on the GPU at the batch sizes the configs name: RWKV-6 7B / batch 16 (the bench workload),
RWKV-6 3B / batch 1, RWKV-7 2.9B / batch 8.  Engine (through the C ABI) vs the C/OpenMP oracle on the same seeded
synthetic `.st`, both activation contracts, with the oracle-vs-oracle distance of the same step beside it.

What is asserted (north_star: logits within 1e-3 relative, argmax exact):
  * default engine path (projection inputs rounded to f16, the web-rwkv fp16 contract): two correct implementations of
    that contract are 2e-3..5e-3 apart at 24-32 layers (oracle/noise_floor.py), so the bound is the measured
    floor of the same step (C oracle f16-contract vs f32-contract), not a constant: engine-vs-oracle <= 2 x floor, and
    the argmax equals the oracle's unless the oracle's own top-2 gap is inside that noise;
  * exact path (split hi+lo f16 operands, no activation rounding): <= 1e-3 against the pure-f32 oracle and argmax exact.
Measured distances are printed as one JSON line per step.
Size-independent properties (determinism, batching invariance, state round trip) run at the 7B shape.
"""
import dataclasses
import json
import os

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth
from oracle import ref_c
from oracle import rwkv_numpy as O

pytestmark = pytest.mark.gpu

if not os.path.exists(ref_c.LIB_PATH):
    from ai00_server_b200 import build
    build.build_oracle()


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def top2_gap(row):
    top = np.partition(row, -2)[-2:]
    return float(top[1] - top[0]) / float(np.abs(row).max())


def make_model(st, B, exact):
    return runtime.Model(st, max_batch=B, token_chunk_size=32, exact=exact)


@pytest.fixture(scope="module")
def big():
    st = synth.make_st("v6-7b", 0)
    m = runtime.Model(st, max_batch=16, token_chunk_size=32)
    yield m, st
    m.close()


def test_full_size_decode_is_deterministic_and_batch_invariant(big):
    m, _ = big
    rng = np.random.default_rng(17)
    zero = m.state.init()
    toks = rng.integers(1, 60000, size=(3, 16))

    def run(slots):
        for s in slots:
            m.state.load(zero, s)
        out = None
        for i in range(3):
            out = m.infer_raw(slots, [1] * len(slots), toks[i, slots].tolist(), [capi.OPTION_LAST] * len(slots))
        return {s: out[j].copy() for j, s in enumerate(slots)}

    a = run(list(range(16)))
    b = run(list(range(16)))
    for s in range(16):
        assert np.array_equal(a[s], b[s])                  # same inputs, same bits
        assert np.isfinite(a[s]).all()
    c = run([2, 9])                                         # two slots alone: same step shape, other slots absent
    assert np.array_equal(c[2], a[2]) and np.array_equal(c[9], a[9])


def test_full_size_state_roundtrip(big):
    m, _ = big
    rng = np.random.default_rng(18)
    m.state.load(m.state.init(), 1)
    m.infer_raw([1], [5], rng.integers(1, 60000, size=5).tolist(), [capi.OPTION_LAST])
    st = m.state.back(1)
    assert np.isfinite(st).all() and np.abs(st).max() > 0
    m.state.load(st, 3)
    assert np.array_equal(m.state.back(3), st)              # load o back = id
    t = int(rng.integers(1, 60000))
    x = m.infer_raw([1], [1], [t], [capi.OPTION_LAST])[0]
    y = m.infer_raw([3], [1], [t], [capi.OPTION_LAST])[0]
    assert np.array_equal(x, y)                             # a restored state continues identically


@pytest.mark.parametrize("preset,B", [("v6-7b", 16), ("v6-3b", 1), ("v7-2b9", 8)])
def test_full_size_parity_with_the_oracle(preset, B):
    st = synth.make_st(preset, 0)
    w = O.parse_st(st)
    c16, c32 = ref_c.RefC(w, "f16"), ref_c.RefC(w, "f32")
    s16, s32 = c16.state_init(B), c32.state_init(B)
    engines = {"default": make_model(st, B, False), "exact": make_model(st, B, True)}
    try:
        for m in engines.values():
            for s in range(B):
                m.state.load(m.state.init(), s)
        rng = np.random.default_rng(19)
        slots = list(range(B))
        prompt = rng.integers(1, 60000, size=(B, 3))
        # a 3-token prompt per slot through the prefill path (one call), token by token in the oracle
        for m in engines.values():
            m.infer_raw(slots, [3] * B, prompt.reshape(-1).tolist(), [capi.OPTION_NONE] * B)
        for j in range(3):
            c16.decode_step(prompt[:, j], s16)
            c32.decode_step(prompt[:, j], s32)
        for i in range(3):
            toks = rng.integers(1, 60000, size=B)
            a, b = c16.decode_step(toks, s16), c32.decode_step(toks, s32)
            floor = rel(a, b)                               # what f16 operand rounding alone does at this depth
            gaps = np.array([top2_gap(r) for r in b])
            rec = {"preset": preset, "batch": B, "step": i, "oracle_f16_vs_f32": floor, "min_top2_gap": float(gaps.min())}
            for name, m in engines.items():
                rows = np.concatenate(m.infer_raw(slots, [1] * B, toks.tolist(), [capi.OPTION_LAST] * B))
                e16, e32 = rel(rows, a), rel(rows, b)
                per_row = np.abs(rows - b).max(1) / np.abs(b).max()
                am16, am32 = rows.argmax(1) == a.argmax(1), rows.argmax(1) == b.argmax(1)
                rec[name] = {"vs_f16_contract": e16, "vs_f32_contract": e32, "argmax_eq_f16": int(am16.sum()),
                             "argmax_eq_f32": int(am32.sum())}
                if name == "exact":
                    assert e32 <= 1e-3, (preset, i, e32)
                    assert am32.all(), (preset, i, np.where(~am32)[0].tolist(), gaps[~am32].tolist())
                else:
                    bound = max(1e-3, 2.0 * floor)
                    assert e16 <= bound and e32 <= bound, (preset, i, e16, e32, floor)
                    # argmax: equal, or the oracle's two best logits of that row are closer than the row's error
                    bad = ~am32 & (gaps > 2.0 * per_row)
                    assert not bad.any(), (preset, i, np.where(bad)[0].tolist())
            print(json.dumps(rec))
    finally:
        for m in engines.values():
            m.close()


def test_front_half_kernel_with_the_7b_lora_rank_matches_the_oracle():
    """The RWKV-6 front-half kernel is templated on the ddlerp LoRA rank: 32 (every CI preset) and 64 (only the 7B shape).
    A 4-layer model with rank 64 puts the 7B instantiation under the 1e-3 bound of the small-model tests."""
    shp = dataclasses.replace(synth.PRESETS["small6"], Dm=64, Dd=128)
    st = synth.make_st(shp, 0)
    m = runtime.Model(st, max_batch=4, token_chunk_size=32)
    try:
        orc = O.Oracle(O.parse_st(st), "f16")
        rng = np.random.default_rng(23)
        counts = [1, 3, 1]
        sts = [orc.state_init() for _ in counts]
        for s in range(3):
            m.state.load(m.state.init(), s)
        for _ in range(4):
            toks = [rng.integers(1, 2000, size=n).tolist() for n in counts]
            rows = m.infer_raw([0, 1, 2], counts, sum(toks, []), [capi.OPTION_LAST] * 3)
            for s in range(3):
                want, sts[s] = orc.run(toks[s], sts[s])
                err = float(np.abs(rows[s] - want).max() / np.abs(want).max())
                assert err <= 1e-3 and rows[s].argmax() == want.argmax(), (s, err)
    finally:
        m.close()
