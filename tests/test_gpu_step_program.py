"""The launches of a step, held to a schedule computed from the model shape alone (DESIGN.md §4, step schedule).

Per layer, a step runs
  * decode-shaped steps (<= 16 tokens) of an RWKV-6 model whose ddlerp LoRA fits pre6_kernel (rank 32 or 64, C % 128 == 0):
    the front half (LN1 + token shift + both LoRA stages) as one launch;
    every other step: LN1, and for RWKV-6 the LoRA W1 and W2 projections;
  * the projections between LN1 and WKV: R/K/V/G with the decay LoRA stage 1 (RWKV-6; as an f16 launch and a quantised one
    in quantised layers), R/K/V with the four adapters' first stages (RWKV-7, split the same way) and the adapters' second
    stages; the RWKV-6 decay LoRA stage 2 only when the WKV kernel cannot fold it (Dd > 128 or Dd % 8 != 0);
  * WKV, O, LN2, the channel-mix key (+ receptance), the channel-mix value.
Around the layers: embedding + LN0 and ln_out, and with output rows the head and the kept-row copy.

Checked: the ordered (type, bytes) list of profile_insitu for a decode step (type 0 LN, 2 WKV, 6 front half, 1000000 + MiB
for a projection, whose bytes are its algorithmic weight bytes: n k 2 for f16, codes + block parameters when quantised), the
launch count of every other step bucket, and profile_step's weight bytes against the decode list."""
import dataclasses

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

SLOTS = [0, 1, 2]
QUANT_LAYERS = 2

# id: (preset, shape overrides, exact, quant_type)
CONFIGS = {
    "small6": ("small6", {}, False, None),                  # front half, decay fold
    "small6-Dd192": ("small6", dict(Dd=192), False, None),  # decay LoRA stage 2 as its own launch on every step
    "small6-Dm16": ("small6", dict(Dm=16), False, None),    # no front half: LN1 + W1 + W2 on every step
    "tiny5": ("tiny5", {}, False, None),
    "tiny7": ("tiny7", {}, False, None),
    "small6-exact": ("small6", {}, True, None),
    "small6-int8": ("small6", {}, False, "int8"),
    "tiny7-int8": ("tiny7", {}, False, "int8"),
}


def f16(n, k):
    return 2 * n * k


def quant(qt):
    """Weight bytes of an [n, k] projection matrix of a layer quantised as `qt` (None: f16; Int8: codes + f16 scale / min
    per 128 inputs)."""
    return f16 if qt is None else (lambda n, k: n * k + n * (k // 128) * 4)


def proj(nbytes):
    return (1000000 + (nbytes >> 20), nbytes)


LN, WKV, PRE6 = (0, 0), (2, 0), (6, 0)


def layer_launches(s, l, decode, qt):
    """The launches of layer l in order, as (type, bytes)."""
    C, F = s.C, s.F
    q = quant(qt)
    out = []
    if s.version == 6:
        if decode and s.Dm in (32, 64) and C % 128 == 0 and C <= 4096:
            out.append(PRE6)
        else:
            out += [LN, proj(f16(5 * s.Dm, C)), proj(5 * f16(C, s.Dm))]
        if qt:
            out += [proj(f16(s.Dd, C)), proj(4 * q(C, C))]
        else:
            out.append(proj(4 * f16(C, C) + f16(s.Dd, C)))
        if not (s.Dd <= 128 and s.Dd % 8 == 0):
            out.append(proj(f16(C, s.Dd)))
    elif s.version == 5:
        out += [LN, proj(4 * q(C, C))]
    else:
        ranks = [s.Dd, s.Da] + ([s.Dv] if l > 0 else []) + [s.Dg]
        first = sum(f16(r, C) for r in ranks)
        out.append(LN)
        out += [proj(first), proj(3 * q(C, C))] if qt else [proj(3 * f16(C, C) + first)]
        out.append(proj(sum(f16(C, r) for r in ranks)))
    out += [WKV, proj(q(C, C)), LN]
    out.append(proj(q(F, C) + (q(C, C) if s.version != 7 else 0)))
    out.append(proj(q(C, F)))
    return out


def traced_schedule(s, decode, qt):
    """Every launch of a step that writes in-situ stamps: the layers and the head."""
    out = []
    for l in range(s.L):
        out += layer_launches(s, l, decode, qt if l < QUANT_LAYERS else None)
    return out + [proj(f16(s.V, s.C))]


def step_launches(s, T, R, qt):
    """Kernel launches of one step of T tokens and R output rows: embedding + LN0, the layers, ln_out, head + kept rows."""
    layers = len(traced_schedule(s, T <= 16, qt)) - 1
    return 1 + layers + 1 + (2 if R > 0 else 0)


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(name):
        if name not in cache:
            preset, over, exact, qt = CONFIGS[name]
            shp = dataclasses.replace(synth.PRESETS[preset], **over)
            st = synth.make_st(shp, 0)
            kw = dict(quant=QUANT_LAYERS, quant_type="Int8") if qt else {}
            m = runtime.Model(st, max_batch=4, token_chunk_size=128, exact=exact, **kw)
            for slot in SLOTS:
                m.state.load(m.state.init(), slot)
            cache[name] = (m, shp, exact, qt)
        return cache[name]

    yield get
    for m, *_ in cache.values():
        m.close()


@pytest.mark.parametrize("name", list(CONFIGS))
def test_decode_step_runs_the_planned_launches(models, name):
    m, s, _, qt = models(name)
    windows, _ = m.profile_insitu(SLOTS, np.array([5, 9, 33], np.uint32), reps=1)
    got = [(w["type"], w["bytes"]) for w in windows]
    assert got == traced_schedule(s, True, qt)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_profile_step_counts_the_bytes_the_decode_step_streams(models, name):
    m, s, _, qt = models(name)
    _, _, nbytes = m.profile_step(SLOTS, np.array([5, 9, 33], np.uint32))
    assert nbytes == sum(b for t, b in traced_schedule(s, True, qt) if t >= 1000000)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_every_step_bucket_launches_the_planned_count(models, name):
    m, s, exact, qt = models(name)
    rng = np.random.default_rng(4)
    cap = 16 if exact else 128              # precision 1 runs every step decode-shaped

    def launches(slots, ntok, option):
        before = m.launch_count()
        m.infer_raw(slots, ntok, rng.integers(1, s.V, size=sum(ntok)).tolist(), [option] * len(slots))
        return m.launch_count() - before

    n = len(SLOTS)
    assert launches(SLOTS, [1] * n, capi.OPTION_LAST) == step_launches(s, n, n, qt)
    assert launches(SLOTS, [1] * n, capi.OPTION_NONE) == step_launches(s, n, 0, qt)
    for T in (17, 33, 65):
        steps = [min(cap, T - t0) for t0 in range(0, T, cap)]
        want = sum(step_launches(s, t, int(i == len(steps) - 1), qt) for i, t in enumerate(steps))
        assert launches([0], [T], capi.OPTION_LAST) == want, T
