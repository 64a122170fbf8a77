"""The pieces of tensor parallelism that a one-GPU machine can test directly, bit for bit:

A. A rank's state layout (csrc/misc.cuh state_xform_kernel with h0 = rank * Hl, the snapshot record [L][C | Hl*N*N | C]),
   through the public ABI.  Every rank of a world is created in turn on device 0 with b200rwkv_create_tp and never connected:
   state_load / back / read / write and snapshot_load / back need no peer, and no step runs (only infer needs tp_connect, and
   two ranks on one GPU would spin against each other in the step's rendezvous).
     - Expected export of rank r of a state X: mask_r(X) = X with rows 1..64 (WKV) zeroed (+0.0) outside the rank's columns
       [r Cl, (r + 1) Cl); the shift rows 0 and 65 are replicated, kept whole.
     - X: every element's bits distinct (so a misplaced element cannot match by accident), -0.0 and subnormals among them;
       compared as uint32.
B. The vocabulary-shard gather of a step (csrc/sample.cuh keep_rows_kernel) through b200rwkv_op_keep, against NumPy indexing:
   a slot whose entry has a row for its last token gets concat(shard[q][row] for q in ranks); every other slot's kept row
   keeps its bits.
"""
import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

pytestmark = pytest.mark.gpu

N = 64
WORLDS = [(p, w) for p in ("tiny5", "tiny6", "tiny7") for w in (2, 4)] + \
         [(p, w) for p in ("small5", "small6", "small7") for w in (2, 4, 8)]


@pytest.fixture(scope="module")
def images():
    cache = {}

    def get(preset):
        if preset not in cache:
            cache[preset] = synth.make_st(preset, 0)
        return cache[preset]

    return get


# ---- A. a rank's state layout ----

def distinct_state(L, C, k):
    """A state [L, N+2, C] whose elements have pairwise distinct bits, distinct from those of distinct_state(L, C, k') too:
    magnitudes in [0.5, 1) from disjoint ranges of k, random signs, shuffled; plus -0.0 in a shift row and subnormals in shift
    and WKV rows (one in every 64-column head block)."""
    n = L * (N + 2) * C
    rng = np.random.default_rng(1000 + k)
    b = np.uint32(0x3F000000) + np.uint32(k * n) + np.arange(n, dtype=np.uint32)
    assert int(b[-1]) < 0x3F800000
    b |= rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)
    x = rng.permutation(b).reshape(L, N + 2, C)
    x[0, 0, 5] = 0x80000000                                       # -0.0
    x[L - 1, N + 1, 7] = 0x00000003 + 0x100 * k                  # subnormals
    for h in range(C // N):
        x[h % L, 1 + (h * 7) % N, h * N + 3] = (0x00000010 + 0x100 * k + h) | (0x80000000 if h % 2 else 0)
    assert np.unique(x).size == n
    return x.view(np.float32)


def mask(x, r, world):
    C = x.shape[2]
    Cl = C // world
    y = x.copy()
    y[:, 1:N + 1, :r * Cl] = 0.0
    y[:, 1:N + 1, (r + 1) * Cl:] = 0.0
    return y


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(u32(a), u32(b))


@pytest.mark.parametrize("preset,world", WORLDS)
def test_rank_state_layout(images, preset, world):
    st = images(preset)
    s = synth.PRESETS[preset]
    L, C = s.L, s.C
    Cl = C // world
    X = [distinct_state(L, C, k) for k in range(3)]
    exports = []
    for r in range(world):
        m = runtime.Model(st, max_batch=3, token_chunk_size=32, device=0, rank=r, world=world)
        try:
            assert m.state.shape() == (C, N + 2, L, 1)
            # a different state in every slot, read back only after all three are loaded: a slot-stride error cannot hide
            for slot in range(3):
                m.state.load(X[slot], slot)
            for slot in range(3):
                assert same(m.state.back(slot), mask(X[slot], r, world)), (r, slot)
            exports.append(m.state.back(0))

            # import ignores the heads of other ranks: Y differs from X[0] only there, over slot 1's X[1]
            Y = X[0].copy()
            other = distinct_state(L, C, 3)
            foreign = np.ones(C, bool)
            foreign[r * Cl:(r + 1) * Cl] = False
            Y[:, 1:N + 1, foreign] = other[:, 1:N + 1, foreign]
            m.state.load(Y, 1)
            assert same(m.state.back(1), mask(X[0], r, world)), r
            assert same(m.state.back(0), mask(X[0], r, world)) and same(m.state.back(2), mask(X[2], r, world))

            # snapshots: the record a host state becomes, a slot's record, and a record written to another slot
            sn = m.state.snapshot_load(X[2])
            assert same(m.state.snapshot_back(sn), mask(X[2], r, world)), r
            rd = m.state.read(0)
            assert same(m.state.snapshot_back(rd), m.state.back(0)), r
            m.state.write(sn, 1)
            assert same(m.state.back(1), mask(X[2], r, world)), r
            m.state.write(rd, 2)
            assert same(m.state.back(2), mask(X[0], r, world)), r
            assert same(m.state.back(0), mask(X[0], r, world))
            sn.free()
            rd.free()

            # an unconnected rank refuses a step before launching anything, and its states are untouched
            before = m.launch_count()
            with pytest.raises(capi.B200Error) as ei:
                m.infer_raw([0], [1], [1], [capi.OPTION_LAST])
            assert ei.value.code == capi.ERR_INVALID and "not connected" in str(ei.value)
            assert m.launch_count() == before == 0
            for slot, want in ((0, X[0]), (1, X[2]), (2, X[0])):
                assert same(m.state.back(slot), mask(want, r, world)), (r, slot)
        finally:
            m.close()

    # the ranks' exports merged column block by column block, as b200rwkv_state_back merges them (merge_state_columns):
    # the shift rows from rank 0, WKV columns [r Cl, (r + 1) Cl) from rank r
    merged = exports[0].copy()
    for r in range(1, world):
        merged[:, 1:N + 1, r * Cl:(r + 1) * Cl] = exports[r][:, 1:N + 1, r * Cl:(r + 1) * Cl]
    assert same(merged, X[0])


# ---- B. the vocabulary-shard gather ----

S_POOL = 6
STEPS = {   # name: (slots, counts, options) -- R and the rows' tokens differ from the entry count
    "mixed": ([4, 0, 2, 5], [3, 2, 1, 4], [capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_LAST, capi.OPTION_LAST]),
    "rows past 16": ([1, 3, 0], [20, 5, 2], [capi.OPTION_FULL, capi.OPTION_NONE, capi.OPTION_LAST]),
    "no rows": ([2, 4], [3, 1], [capi.OPTION_NONE, capi.OPTION_NONE]),
}


def keep_reference(keep, shards, slots, counts, options):
    """NumPy indexing: the logits row of every entry's last token, if it has one, gathered from the shards in rank order."""
    want = keep.copy()
    row = 0
    for sl, n, o in zip(slots, counts, options):
        rows = n if o == capi.OPTION_FULL else (1 if o == capi.OPTION_LAST else 0)
        if rows:
            want[sl] = np.concatenate([shards[q, row + rows - 1] for q in range(shards.shape[0])])
        row += rows
    return want


def distinct_f32(n, base, rng):
    b = np.uint32(base) + rng.permutation(n).astype(np.uint32)
    return b.view(np.float32)


@pytest.mark.parametrize("world,Vl", [(w, v) for w in (1, 2, 3, 8) for v in (5, 4096, 4097, 4098, 4099, 8192, 8193)] + [(1, 65536)])
@pytest.mark.parametrize("step", list(STEPS))
def test_keep_rows_gathers_every_shard(step, world, Vl):
    """Vl % 4 = 1, 2, 3 put shard rows and destination rows at every 4-byte offset modulo 16 (the float4 / scalar paths and
    the scalar tail), Vl > 2048 runs the KEEP_CHUNKS x KEEP_THREADS float4 loop more than once, and "rows past 16" gives a
    step of 21 logits rows (two 16-row tiles of CTAs)."""
    slots, counts, options = STEPS[step]
    R = sum(n if o == capi.OPTION_FULL else (1 if o == capi.OPTION_LAST else 0) for n, o in zip(counts, options))
    V = world * Vl
    rng = np.random.default_rng(world * 100003 + Vl)
    shards = distinct_f32(world * max(R, 1) * Vl, 0x3F000000, rng).reshape(world, max(R, 1), Vl)[:, :R].copy()
    keep = distinct_f32(S_POOL * V, 0xBF000000, rng).reshape(S_POOL, V)      # sentinels: negative, never in a shard
    want = keep_reference(keep, shards, slots, counts, options)
    capi.op_keep(slots, counts, options, shards, keep)
    assert same(keep, want), [int(np.sum(u32(keep[s]) != u32(want[s]))) for s in range(S_POOL)]
