"""Batch-invariant engines (b200rwkv_options.batch_invariant; DESIGN.md §6): every per-token result of a slot is the bits a
decode step (one token per entry, at most 16 entries) gives it, whatever else shares its calls, whatever token_chunk_size is
and however its tokens are cut into calls.  Every comparison is bit for bit, on the uint32 views."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

LAST, FULL, NONE, SCORE = capi.OPTION_LAST, capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_SCORE

# id: (preset, shape overrides, quant_type)
CONFIGS = {
    "tiny5": ("tiny5", {}, None),
    "tiny6": ("tiny6", {}, None),
    "tiny7": ("tiny7", {}, None),
    "small6": ("small6", {}, None),
    "tiny6-int8": ("tiny6", {}, "Int8"),
    "tiny6-nf4": ("tiny6", {}, "NF4"),
    "tiny7-int8": ("tiny7", {}, "Int8"),
    "tiny7-nf4": ("tiny7", {}, "NF4"),
    "7b-layer": ("v6-7b", dict(L=1, V=4096), None),
}
_ST = {}


def shape(name):
    preset, over, _ = CONFIGS[name]
    return dataclasses.replace(synth.PRESETS[preset], **over)


def model(name, batch_invariant=True, chunk=128, max_batch=8, precision=0):
    if name not in _ST:
        _ST[name] = synth.make_st(shape(name), 0)
    qt = CONFIGS[name][2]
    kw = dict(quant=shape(name).L, quant_type=qt) if qt else {}
    m = runtime.Model(_ST[name], max_batch=max_batch, token_chunk_size=chunk, precision=precision,
                      batch_invariant=batch_invariant, **kw)
    zero = m.state.init()
    for s in range(max_batch):
        m.state.load(zero, s)
    return m


def same(a, b, what=""):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape, what
    bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} differ, first at {np.unravel_index(bad[0], a.shape)}"


def kept_row(m, slot):
    snap = m.state.read(slot)
    try:
        return m.state.snapshot_back(snap, with_logits=True)[1]
    finally:
        snap.free()


def decode(m, slot, toks, hidden_layers=()):
    """The reference: one token per call.  Rows [n, V] and, per layer of hidden_layers, the hidden rows [n, C]."""
    rows, hid = [], {l: [] for l in hidden_layers}
    for t in toks:
        rows.append(m.infer_raw([slot], [1], [int(t)], [LAST])[0][0].copy())
        for l in hidden_layers:
            hid[l].append(m.last_hidden(max_rows=1, layer=l)[0].copy())
    return np.stack(rows), {l: np.stack(v) for l, v in hid.items()}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_long_prompt_matches_token_by_token_decode(name):
    """A 300-token FULL prompt (steps of 128, 128 and 44 tokens) against the same tokens fed one per call: every row, the
    state and the kept row."""
    m = model(name)
    try:
        V = m.info["num_vocab"]
        toks = np.random.default_rng(1).integers(1, V, size=300).tolist()
        full = m.infer_raw([0], [300], toks, [FULL])[0].copy()
        ref, _ = decode(m, 1, toks)
        same(full, ref, "logits rows")
        same(m.state.back(0), m.state.back(1), "state")
        same(kept_row(m, 0), kept_row(m, 1), "kept row")
    finally:
        m.close()


@pytest.mark.parametrize("name", ["tiny6", "tiny7", "small6", "tiny6-int8"])
def test_ragged_neighbours_chunks_and_call_cuts_do_not_move_a_slot(name):
    """One slot's 200 tokens, fed alone one per call, then beside ragged neighbours (1, 17, 40 and 130 tokens, LAST / FULL /
    NONE / SCORE, permuted slots) at chunk 16 / 32 / 64 / 128 and odd call cuts: rows, SCORE values and argmax ids, states,
    recorded and pooled hidden rows."""
    s = shape(name)
    layers = sorted({0, s.L - 1})
    rng = np.random.default_rng(2)
    toks = rng.integers(1, s.V, size=200).tolist()
    ref_m = model(name, chunk=16, max_batch=8)
    try:
        ref_m.keep_hidden(layers=layers)
        ref_rows, ref_hid = decode(ref_m, 0, toks, layers)
        ref_state = ref_m.state.back(0)
        # SCORE one token per call: token j scored from the row of token j - 1 (the kept row for j = 0)
        ref_m.state.load(ref_m.state.init(), 1)
        ref_m.infer_raw([1], [1], [toks[0]], [LAST])
        ref_score = [ref_m.infer_ex([1], [1], [t], [SCORE])[1][0] for t in toks[1:]]
        ref_lp = np.concatenate([a for a, _ in ref_score])
        ref_am = np.concatenate([b for _, b in ref_score])
    finally:
        ref_m.close()

    sizes, opts = [1, 17, 40, 130], [LAST, FULL, NONE, SCORE]
    for chunk, cuts, perm in ((16, [200], 0), (32, [37, 163], 1), (64, [100, 100], 2), (128, [1, 128, 71], 3)):
        m = model(name, chunk=chunk, max_batch=8)
        try:
            m.keep_hidden(layers=layers)
            got_rows, got_hid = [], {l: [] for l in layers}
            pos = 0
            for ci, n in enumerate(cuts):
                nb = np.random.default_rng(10 + ci).permutation(4)
                nslots = [3 + ((int(k) + perm) % 4) for k in nb]
                ents = [(nslots[i], sizes[k], opts[(k + ci + perm) % 4]) for i, k in enumerate(nb)]
                ents.insert((ci + perm) % 5, (0, n, FULL))
                slots = [e[0] for e in ents]
                ntok = [e[1] for e in ents]
                opt = [e[2] for e in ents]
                feed = []
                for sl, nt, _ in ents:
                    feed += toks[pos:pos + n] if sl == 0 else rng.integers(1, s.V, size=nt).tolist()
                rows, _ = m.infer_ex(slots, ntok, feed, opt)
                i0 = slots.index(0)
                got_rows.append(rows[i0].copy())
                t0 = sum(ntok[:i0])
                for l in layers:
                    got_hid[l].append(m.last_hidden(max_rows=sum(ntok), layer=l)[t0:t0 + n].copy())
                pos += n
            same(np.concatenate(got_rows), ref_rows, f"rows chunk {chunk}")
            for l in layers:
                same(np.concatenate(got_hid[l]), ref_hid[l], f"hidden layer {l} chunk {chunk}")
            same(m.state.back(0), ref_state, f"state chunk {chunk}")
            # SCORE over the whole sequence in one entry beside neighbours; pooled rows of the same call
            m.keep_hidden(layers=[])
            m.keep_hidden_pooled([s.L - 1], "last")
            m.state.load(m.state.init(), 1)
            m.infer_raw([1], [1], [toks[0]], [LAST])
            slots, ntok = [6, 1, 4], [40, 199, 17]
            feed = rng.integers(1, s.V, size=40).tolist() + toks[1:] + rng.integers(1, s.V, size=17).tolist()
            _, sc = m.infer_ex(slots, ntok, feed, [FULL, SCORE, NONE])
            same(sc[1][0], ref_lp, f"SCORE values chunk {chunk}")
            assert np.array_equal(sc[1][1], ref_am), f"SCORE argmax chunk {chunk}"
            pooled, _ = m.last_hidden_pooled(s.L - 1, max_rows=3)
            same(pooled[1], ref_hid[s.L - 1][-1], f"pooled last row chunk {chunk}")
            m.keep_hidden_pooled([])
        finally:
            m.close()


@pytest.mark.parametrize("name", ["tiny6", "tiny7", "tiny5"])
def test_wide_decode_matches_each_slot_alone(name):
    """40 slots stepping together (steps of 40 tokens) for 4 tokens against each slot stepping alone."""
    m = model(name, max_batch=41)
    try:
        V = m.info["num_vocab"]
        toks = np.random.default_rng(3).integers(1, V, size=(40, 4))
        for j in range(4):
            wide = m.infer_raw(list(range(40)), [1] * 40, toks[:, j].tolist(), [LAST] * 40)
        for s in range(40):
            m.state.load(m.state.init(), 40)
            for j in range(4):
                alone = m.infer_raw([40], [1], [int(toks[s, j])], [LAST])[0]
            same(wide[s], alone, f"slot {s} row")
            same(m.state.back(s), m.state.back(40), f"slot {s} state")
    finally:
        m.close()


@pytest.mark.parametrize("name", ["tiny6", "tiny7", "small6"])
def test_snapshots_inside_a_long_entry_are_the_decode_states(name):
    """b200rwkv_infer_snapshots inside a 300-token NONE entry: each snapshot's state and row equal the token-by-token state
    and LAST row at that position."""
    m = model(name)
    try:
        V = m.info["num_vocab"]
        toks = np.random.default_rng(4).integers(1, V, size=300).tolist()
        at = [1, 16, 17, 100, 128, 129, 255, 300]
        _, _, snaps = m.infer_snapshots([0], [300], toks, [NONE], [(0, p) for p in at])
        got = [m.state.snapshot_back(sn, with_logits=True) for sn in snaps]
        for sn in snaps:
            sn.free()
        pos = 0
        for (st, lg), p in zip(got, at):
            rows, _ = decode(m, 1, toks[pos:p])
            pos = p
            same(lg, rows[-1], f"snapshot row at {p}")
            same(st, m.state.back(1), f"snapshot state at {p}")
    finally:
        m.close()


@pytest.mark.parametrize("name", ["tiny5", "tiny6", "tiny7", "tiny6-int8"])
def test_short_steps_and_precision_1_are_unchanged(name):
    """Steps of <= 16 tokens on a mode engine against a default engine: same bits, same launches.  With precision 1 the mode
    changes nothing at any shape."""
    shapes = [([0, 1, 2], [1, 1, 1], [LAST] * 3), ([0, 1], [9, 7], [FULL, LAST]), ([3], [16], [FULL])]
    long_shapes = [([0, 1], [30, 50], [FULL, LAST]), ([2], [128], [LAST])]
    for precision in (0, 1):
        if precision and CONFIGS[name][2]:
            continue
        a, b = model(name, precision=precision), model(name, batch_invariant=False, precision=precision)
        try:
            V = a.info["num_vocab"]
            rng = np.random.default_rng(5)
            for slots, ntok, opt in shapes + (long_shapes if precision else []):
                toks = rng.integers(1, V, size=sum(ntok)).tolist()
                n0, n1 = a.launch_count(), b.launch_count()
                ra, rb = a.infer_raw(slots, ntok, toks, opt), b.infer_raw(slots, ntok, toks, opt)
                assert a.launch_count() - n0 == b.launch_count() - n1, (precision, ntok)
                for x, y in zip(ra, rb):
                    same(x, y, f"precision {precision} {ntok}")
                for s in slots:
                    same(a.state.back(s), b.state.back(s), f"precision {precision} {ntok} state")
        finally:
            a.close()
            b.close()


def test_mode_launches_the_planned_count_per_step_bucket():
    """Per layer, a mode step of more than 16 tokens runs the decode step's launches, with an RWKV-6 front half as two
    launches (the wide LN1 and the front half's LoRA phases) instead of one."""
    from test_gpu_step_program import CONFIGS as PROG, QUANT_LAYERS, traced_schedule
    for name in ("small6", "small6-Dd192", "small6-Dm16", "tiny5", "tiny7", "small6-int8"):
        preset, over, _, qt = PROG[name]
        s = dataclasses.replace(synth.PRESETS[preset], **over)
        kw = dict(quant=QUANT_LAYERS, quant_type="Int8") if qt else {}
        m = runtime.Model(synth.make_st(s, 0), max_batch=4, token_chunk_size=128, batch_invariant=True, **kw)
        try:
            m.state.load(m.state.init(), 0)
            front = s.version == 6 and s.Dm in (32, 64) and s.C % 128 == 0 and s.C <= 4096
            per_step = len(traced_schedule(s, True, qt)) - 1 + (s.L if front else 0)
            for T in (17, 33, 65, 128):
                for R, opt in ((1, LAST), (0, NONE)):
                    before = m.launch_count()
                    m.infer_raw([0], [T], np.arange(1, T + 1).tolist(), [opt])
                    assert m.launch_count() - before == 1 + per_step + 1 + (2 if R else 0), (name, T, R)
        finally:
            m.close()


# ---------------------------------------------------------------------------------------------------------------------
# op level
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("quant", [capi.QUANT_NONE, capi.QUANT_INT8, capi.QUANT_NF4])
def test_forced_grid_gemm_gives_each_token_the_bits_of_a_16_token_launch(quant):
    """A wgmma with N = 128 gives every output element the bits of N = 16 at the same K split: op_gemm with a forced grid
    (grid_wide = grid) over 128 tokens against the same rows in launches of 16, every act and out_mode."""
    rng = np.random.default_rng(6)
    N, K, grid = 384, 1024, 10          # 3 tiles x 8 k blocks over 10 CTAs: every tile cut
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((1, 128, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    xx, sx = rng.standard_normal((1, 128, N)).astype(np.float32), rng.standard_normal((1, 128, N)).astype(np.float32)
    mu = rng.random(N).astype(np.float32)
    acts = range(capi.ACT_V7DECAY + 1) if quant == capi.QUANT_NONE else [capi.ACT_NONE, capi.ACT_TANH]
    cases = [(a, capi.OUT_F32) for a in acts] + [(capi.ACT_TANH, capi.OUT_A16), (capi.ACT_NONE, capi.OUT_LERP_A16)]
    for act, mode in cases:
        def run(T, t0):
            rows = capi.gemm_rows(T)
            dt = np.float32 if mode == capi.OUT_F32 else np.uint16
            d = dict(w=w, x=x[:, t0:t0 + T], act=act, out_mode=mode, out=np.zeros((1, rows, N), dt))
            if mode == capi.OUT_F32:
                d["bias"] = bias
            if mode == capi.OUT_LERP_A16:
                d.update(xx=xx[:, t0:t0 + T], sx=sx[:, t0:t0 + T], mu=mu)
            capi.op_gemm(T, [d], quant_type=quant, grid=grid)
            return d["out"][0, :T]
        wide = run(128, 0)
        narrow = np.concatenate([run(16, t0) for t0 in range(0, 128, 16)])
        assert np.array_equal(wide.view(np.uint16 if wide.dtype == np.uint16 else np.uint32),
                              narrow.view(np.uint16 if narrow.dtype == np.uint16 else np.uint32)), (act, mode)


def ln_case(stage, T, C, S, rng, Dm=32):
    """Arrays of one op_ln step of T one-token entries (slots 0..T-1) of C channels."""
    a = dict(S=S, x_in=rng.standard_normal((1, T, C)).astype(np.float32), ln_w=(1 + 0.1 * rng.standard_normal(C)).astype(np.float32),
             ln_b=(0.1 * rng.standard_normal(C)).astype(np.float32), shift_state=rng.standard_normal((S, C)).astype(np.float32),
             n_parts=2, parts=rng.standard_normal((1, 2, T, C)).astype(np.float32),
             commit_src=rng.standard_normal((1, T, C)).astype(np.float32), commit_dst=np.zeros((S, C), np.float32),
             hidden=np.zeros((1, T, C), np.float32), x_out=np.zeros((1, T, C), np.float32),
             xx_out=np.zeros((1, T, C), np.float32), sx_out=np.zeros((1, T, C), np.float32))
    n_mix = 1 if stage == capi.LN_FRONT6 else 4
    a.update(n_mix=n_mix, mu=rng.random((n_mix, C)).astype(np.float32))
    if stage == capi.LN_FRONT6:
        a.update(Dm=Dm, W1=(0.05 * rng.standard_normal((5 * Dm, C))).astype(np.float16).view(np.uint16),
                 W2=(0.05 * rng.standard_normal((5, C, Dm))).astype(np.float16).view(np.uint16),
                 mu5=rng.random((5, C)).astype(np.float32))
    return a


def ln_run(stage, a, slots, T, bi):
    rows = capi.gemm_rows(T)
    b = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in a.items()}
    C = b["x_in"].shape[2]
    b["mix_out"] = np.zeros((1, b["n_mix"], rows, C), np.uint16)
    if stage == capi.LN_FRONT6:
        b["lora_out"] = np.zeros((1, 5, rows, b["Dm"]), np.uint16)
        b["out5"] = np.zeros((1, 5, rows, C), np.uint16)
    kern = capi.op_ln(stage, C, slots, [1] * len(slots), batch_invariant=bi, **b)
    return b, kern


@pytest.mark.parametrize("stage", [capi.LN_MIX, capi.LN_FRONT6])
@pytest.mark.parametrize("T", [17, 33, 100, 128])
def test_wide_ln_stages_give_each_row_the_decode_kernels_bits(stage, T):
    """op_ln with batch_invariant over T one-token entries against the same entries in steps of <= 16 (the cluster kernel /
    pre6_kernel): every output row, bit for bit."""
    C, S = 512, 128
    rng = np.random.default_rng(T)
    a = ln_case(stage, T, C, S, rng)
    wide, kern = ln_run(stage, a, list(range(T)), T, True)
    assert kern[0] == (capi.K_PRE6_WIDE if stage == capi.LN_FRONT6 else capi.K_LN_MIX_CLUSTER_WIDE)
    for t0 in range(0, T, 16):
        n = min(16, T - t0)
        sub = {k: (v[:, t0:t0 + n] if k in ("x_in", "commit_src", "hidden", "x_out", "xx_out", "sx_out") else v)
               for k, v in a.items()}
        sub["parts"] = a["parts"][:, :, t0:t0 + n]
        sub = {k: (np.ascontiguousarray(v) if isinstance(v, np.ndarray) else v) for k, v in sub.items()}
        narrow, k16 = ln_run(stage, sub, list(range(t0, t0 + n)), n, False)
        assert k16[0] == (capi.K_PRE6 if stage == capi.LN_FRONT6 else capi.K_LN_MIX_CLUSTER)
        for key in ("x_out", "xx_out", "sx_out", "hidden"):
            same(wide[key][:, t0:t0 + n], narrow[key], f"{key} rows {t0}..")
        outs = ("mix_out",) + (("lora_out", "out5") if stage == capi.LN_FRONT6 else ())
        for key in outs:
            assert np.array_equal(wide[key][..., t0:t0 + n, :], narrow[key][..., :n, :]), f"{key} rows {t0}.."
        rows = list(range(t0, t0 + n))
        same(wide["commit_dst"][rows], narrow["commit_dst"][rows], f"commit rows {t0}..")
