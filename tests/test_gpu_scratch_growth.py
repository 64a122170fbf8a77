"""Run-time buffers regrown in the middle of an engine's life.  The softmax rows, the sample_probs rows, the sample_topk
staging blob, the SCORE rows and the recorded hidden rows (keep_hidden, keep_hidden_layers) are allocated on first use and
grown when a later call needs more.  One engine drives each of them below its first size, past it and below it again; every
call gives the same bits as the same call on a freshly created engine of the same model."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

V = 65536                 # the World vocabulary: one probability row is 256 KiB, so four fill the first 1 MiB block
MAX_BATCH = 16


@pytest.fixture(scope="module")
def st():
    return synth.make_st(dataclasses.replace(synth.PRESETS["tiny6"], V=V), 0)


def new_model(st):
    return runtime.Model(st, max_batch=MAX_BATCH, token_chunk_size=128)


@pytest.fixture(scope="module")
def engine(st):
    m = new_model(st)
    yield m
    m.close()


def check_sizes(engine, st, sizes, call):
    """call(model, size) -> list of arrays: on the long-lived engine the same bits as on a fresh engine, size after size."""
    for n in sizes:
        got = call(engine, n)
        fresh = new_model(st)
        try:
            want = call(fresh, n)
        finally:
            fresh.close()
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert g.shape == w.shape and np.array_equal(g.view(np.uint32), w.view(np.uint32)), n


def keep_rows(m, slots):
    """Fresh states and two tokens per slot with a LAST row: every slot holds a kept logits row."""
    for s in slots:
        m.state.load(m.state.init(), s)
    toks = [t for s in slots for t in (s + 1, 2 * s + 5)]
    m.infer_raw(slots, [2] * len(slots), toks, [capi.OPTION_LAST] * len(slots), keep_on_device=True)


def test_softmax_rows(engine, st):
    def call(m, rows):
        x = np.random.default_rng(rows).standard_normal((rows, V)).astype(np.float32)
        return m.softmax(list(x))

    check_sizes(engine, st, (1, 70, 1), call)


def test_sample_probs_rows(engine, st):
    """Eight rows need 2 MiB, past the first block of 1 MiB."""
    def call(m, nrows):
        slots = list(range(nrows))
        keep_rows(m, slots)
        return [m.sample_probs(slots)]

    check_sizes(engine, st, (1, 8, 1), call)


def test_sample_topk_staging(engine, st):
    """Two rows of 40000 penalties and 40000 biases each stage 1.28 MB of lists, past the first 1 MiB blob."""
    def call(m, n):
        rng = np.random.default_rng(n)
        slots = [0, 1]
        keep_rows(m, slots)
        pen = [dict(zip(rng.choice(V, n, replace=False).tolist(), rng.random(n).tolist())) for _ in slots]
        bias = [dict(zip(rng.choice(V, n, replace=False).tolist(), (rng.random(n) - 0.5).tolist())) for _ in slots]
        return list(m.sample_topk(slots, penalties=pen, bias=bias, top_k=64))

    check_sizes(engine, st, (5, 40000, 5), call)


def test_score_rows(engine, st):
    """300 scored tokens in one call: past the first block of 256 rows."""
    def call(m, n):
        keep_rows(m, [0])
        toks = np.random.default_rng(n).integers(1, 500, size=n).tolist()
        _, sc = m.infer_ex([0], [n], toks, [capi.OPTION_SCORE])
        return list(sc[0])

    check_sizes(engine, st, (5, 300, 5), call)


def test_hidden_rows(engine, st):
    """300 tokens in one call, recorded after the last layer and after each chosen layer: past the first 256 rows."""
    def call(m, n):
        toks = np.random.default_rng(n).integers(1, 500, size=n).tolist()
        m.keep_hidden(True)
        m.keep_hidden(layers=[1, 0])
        try:
            m.state.load(m.state.init(), 0)
            m.infer_raw([0], [n], toks, [capi.OPTION_NONE])
            rows = [m.last_hidden(max_rows=n)] + [m.last_hidden(max_rows=n, layer=layer) for layer in (1, 0)]
        finally:
            m.keep_hidden(False)
            m.keep_hidden(layers=[])
        assert all(r.shape == (n, m.info["num_emb"]) for r in rows)
        return rows

    check_sizes(engine, st, (5, 300, 5), call)
