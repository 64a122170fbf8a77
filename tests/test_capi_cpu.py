"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the
header declares, the host-only entry points work, and device entry points fail loudly (there
is no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ai00_server_b200 import capi, runtime, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_library_exports_exactly_the_declared_symbols():
    import shutil
    import subprocess
    hdr = open(os.path.join(ROOT, "include", "b200rwkv.h")).read()
    declared = set(re.findall(r"\b(b200rwkv_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"b200rwkv_status", "b200rwkv_info", "b200rwkv_engine", "b200rwkv_options"}
    assert len(declared) >= 30
    lib = capi.lib()
    bound = {n for n, _, _ in capi.SYMBOLS}
    assert declared == bound, (declared ^ bound)
    for name in declared:
        assert getattr(lib, name) is not None
    # and nothing else: the removed HBM-streaming / L2-prefetch micro-benchmark entries in particular
    for name in ("b200rwkv_debug_stream", "b200rwkv_debug_prefetch"):
        assert not hasattr(lib, name)
    nm = shutil.which("nm")
    if nm is not None:
        out = subprocess.run([nm, "-D", "--defined-only", capi.LIB_PATH], check=True, capture_output=True, text=True).stdout
        exported = {f[-1] for f in (l.split() for l in out.splitlines()) if f and f[-1].startswith("b200rwkv_")}
        assert exported == declared, (exported ^ declared)


def test_product_library_ignores_the_environment():
    """The library reads no environment variable (the CUDA runtime linked into it reads its own CUDA_* variables): no engine
    source calls getenv, and no source or build recipe names a B200RWKV_DEBUG macro that could compile a switch back in."""
    csrc = os.path.join(ROOT, "ai00_server_b200", "csrc")
    sources = [os.path.join(csrc, f) for f in sorted(os.listdir(csrc))]
    sources += [os.path.join(ROOT, "include", f) for f in sorted(os.listdir(os.path.join(ROOT, "include")))]
    sources.append(os.path.join(ROOT, "ai00_server_b200", "build.py"))
    for path in sources:
        src = open(path, errors="replace").read()
        if path.startswith(csrc):
            assert "getenv(" not in src, path
        assert "B200RWKV_DEBUG" not in src, path


def test_info_from_st_host_only():
    for preset, ver in (("tiny5", 5), ("tiny6", 6), ("tiny7", 7)):
        info = capi.info_from_st(synth.make_st(preset, 0))
        s = synth.PRESETS[preset]
        assert info["version"] == ver
        assert (info["num_layer"], info["num_emb"], info["num_hidden"], info["num_vocab"]) == (s.L, s.C, s.F, s.V)
        assert (info["num_head"], info["head_size"]) == (s.H, 64)
    i6 = capi.info_from_st(synth.make_st("tiny6", 0))
    assert (i6["time_mix_adapter"], i6["time_decay_adapter"]) == (32, 64)


def test_malformed_st_is_an_error_not_a_crash():
    junk = np.frombuffer(b"\x10\x00\x00\x00\x00\x00\x00\x00{\"a\":1}        ", dtype=np.uint8).copy()
    with pytest.raises(capi.B200Error) as ei:
        capi.info_from_st(junk)
    assert ei.value.code == capi.ERR_INVALID
    with pytest.raises(capi.B200Error):
        capi.info_from_st(np.zeros(4, np.uint8))


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_create_fails_loudly_without_gpu():
    with pytest.raises(capi.B200Error) as ei:
        runtime.Model(synth.make_st("tiny6", 0), max_batch=2, token_chunk_size=16)
    assert ei.value.code == capi.ERR_CUDA
    assert "no CPU fallback" in str(ei.value)


def test_bad_precision_rejected():
    """precision 0 = f16 activations, 1 = f32-exact activations (web-rwkv Bundle::<f32>); anything else is invalid."""
    st = synth.make_st("tiny6", 0)
    h = C.c_void_p()
    code = capi.lib().b200rwkv_create(capi.ptr(st), st.size, 0, 2, 16, 7, C.byref(h))
    assert code == capi.ERR_INVALID
    assert not h.value


def _edit_header(st: np.ndarray, fn) -> np.ndarray:
    import json
    import struct
    raw = st.tobytes()
    hlen = struct.unpack("<Q", raw[:8])[0]
    hdr = json.loads(raw[8:8 + hlen])
    fn(hdr)
    h2 = json.dumps(hdr, separators=(",", ":")).encode()
    return np.frombuffer(struct.pack("<Q", len(h2)) + h2 + raw[8 + hlen:], dtype=np.uint8).copy()


def test_st_tensor_sizes_are_validated():
    """A tensor whose byte range does not equal dtype x shape, a wrong rank, or an absurd shape must be a clean
    B200RWKV_ERR_INVALID from the host-only parser (ADVICE r1: the loader trusted shape-derived sizes)."""
    st = synth.make_st("tiny6", 0)
    assert capi.info_from_st(st)["version"] == 6

    def short_tensor(h):
        b, e = h["blocks.0.att.key.weight"]["data_offsets"]
        h["blocks.0.att.key.weight"]["data_offsets"] = [b, e - 64]

    def huge_shape(h):
        h["emb.weight"]["shape"] = [1 << 40, 1 << 40]

    def wrong_rank(h):
        t = h["blocks.0.att.time_first"]
        t["shape"] = [int(np.prod(t["shape"]))]

    def bad_dtype(h):
        h["emb.weight"]["dtype"] = "Q7"

    def deep_metadata(h):
        node = cur = {}
        for _ in range(200):
            cur["x"] = {}
            cur = cur["x"]
        h["__metadata__"] = node

    for fn in (short_tensor, huge_shape, wrong_rank, bad_dtype, deep_metadata):
        with pytest.raises(capi.B200Error) as ei:
            capi.info_from_st(_edit_header(st, fn))
        assert ei.value.code == capi.ERR_INVALID, fn.__name__


def test_runtime_chunking_bookkeeping():
    """Runtime.infer mirrors web-rwkv: <= token_chunk_size tokens per call, Last rows only once a
    slot's run is exhausted (reference run.rs:1134-1155).  Engine calls are stubbed."""
    calls = []

    class Stub:
        info = {"num_vocab": 8}

        def infer_raw(self, slots, ntok, toks, opts):
            calls.append((list(slots), list(ntok), list(toks), list(opts)))
            return [np.zeros((nt if o == capi.OPTION_FULL else (1 if o == capi.OPTION_LAST else 0), 8), np.float32)
                    for nt, o in zip(ntok, opts)]

    rt = runtime.Runtime(Stub())
    inp = runtime.RnnInput([runtime.RnnInputBatch([1, 2, 3, 4, 5], runtime.RnnOption.Last),
                            runtime.RnnInputBatch([], runtime.RnnOption.Last),
                            runtime.RnnInputBatch([7, 8], runtime.RnnOption.Full)], 4)
    seen_rows = {0: 0, 2: 0}
    while inp.num_token() > 0:
        inp, out = rt.infer(inp)
        for b, o in enumerate(out):
            if not o.is_empty():
                seen_rows[b] += o.data.shape[0]
    assert seen_rows == {0: 1, 2: 2}
    assert calls[0] == ([0], [4], [1, 2, 3, 4], [capi.OPTION_NONE])
    assert calls[1] == ([0, 2], [1, 2], [5, 7, 8], [capi.OPTION_LAST, capi.OPTION_FULL])


def test_read_state_host_only():
    """`vN::read_state` (reference lib.rs:378-389): a state-tuned model / `.state` file -> the [L, N+2, C] state tensor; the
    oracle builds the same tensor from the same file (row 1+i, column h*N+j <- time_state[h][i][j])."""
    import dataclasses
    import json
    import struct
    from oracle import rwkv_numpy as O
    shp = dataclasses.replace(synth.PRESETS["tiny6"], time_state=True)
    st = synth.make_st(shp, 0)
    info = capi.info_from_st(st)
    got = runtime.read_state(info, st)
    want = O.Oracle(O.parse_st(st), "f16").state_init()
    assert got.shape == want.shape and np.array_equal(got, want) and np.abs(got[:, 1:65]).max() > 0
    assert np.all(got[:, 0] == 0) and np.all(got[:, 65] == 0)
    # a stand-alone `.state` file: only the time_state tensors, stored as F32
    w = O.parse_st(st)
    names = [n for n in w if n.endswith("att.time_state")]
    hdr, blobs, off = {"__metadata__": {"format": "pt"}}, [], 0
    for n in names:
        b = w[n].astype(np.float32).tobytes()
        hdr[n] = {"dtype": "F32", "shape": list(w[n].shape), "data_offsets": [off, off + len(b)]}
        blobs.append(b); off += len(b)
    h = json.dumps(hdr).encode()
    img = np.frombuffer(struct.pack("<Q", len(h)) + h + b"".join(blobs), np.uint8).copy()
    assert np.array_equal(runtime.read_state(info, img), want)
    with pytest.raises(capi.B200Error) as ei:           # a model without time_state is not a state file
        runtime.read_state(info, synth.make_st("tiny6", 0))
    assert ei.value.code == capi.ERR_INVALID


def test_ctypes_structs_match_the_header(tmp_path):
    """The ctypes mirrors of the two ABI structs have the layout a C compiler gives include/b200rwkv.h (a plain C translation unit:
    the header must stay C, not C++)."""
    import ctypes as C
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200rwkv.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b200rwkv_options), offsetof(b200rwkv_options, devices),\n'
                   '  offsetof(b200rwkv_options, lora_st), offsetof(b200rwkv_options, quant_layers), sizeof(b200rwkv_info),\n'
                   '  sizeof(b200rwkv_gemm_seg), offsetof(b200rwkv_gemm_seg, act), offsetof(b200rwkv_gemm_seg, lerp_xx),\n'
                   '  offsetof(b200rwkv_gemm_seg, out));\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b200rwkv_wkv_args), offsetof(b200rwkv_wkv_args, slot),\n'
                   '  offsetof(b200rwkv_wkv_args, precision), offsetof(b200rwkv_wkv_args, r), offsetof(b200rwkv_wkv_args, nu),\n'
                   '  offsetof(b200rwkv_wkv_args, layer0), offsetof(b200rwkv_wkv_args, v_first), offsetof(b200rwkv_wkv_args, Dd),\n'
                   '  offsetof(b200rwkv_wkv_args, out));\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", offsetof(b200rwkv_wkv_args, nsnap), offsetof(b200rwkv_wkv_args, snap_tok),\n'
                   '  offsetof(b200rwkv_wkv_args, snap_rec), offsetof(b200rwkv_wkv_args, snap_ld), offsetof(b200rwkv_wkv_args, snap_off));\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b200rwkv_ln_args), offsetof(b200rwkv_ln_args, slot),\n'
                   '  offsetof(b200rwkv_ln_args, precision), offsetof(b200rwkv_ln_args, x_in), offsetof(b200rwkv_ln_args, parts),\n'
                   '  offsetof(b200rwkv_ln_args, n_mix), offsetof(b200rwkv_ln_args, mix_out), offsetof(b200rwkv_ln_args, Dm),\n'
                   '  offsetof(b200rwkv_ln_args, V), offsetof(b200rwkv_ln_args, kernel_out));\n'
                   '  printf("%zu %zu %zu %zu %zu %zu\\n", offsetof(b200rwkv_ln_args, nsnap), offsetof(b200rwkv_ln_args, snap_tok),\n'
                   '  offsetof(b200rwkv_ln_args, snap_rec), offsetof(b200rwkv_ln_args, snap_ld), offsetof(b200rwkv_ln_args, snap_off),\n'
                   '  offsetof(b200rwkv_ln_args, snap_head_out));\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(b200rwkv_keep_args), offsetof(b200rwkv_keep_args, slot),\n'
                   '  offsetof(b200rwkv_keep_args, world), offsetof(b200rwkv_keep_args, shards), offsetof(b200rwkv_keep_args, keep));\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b200rwkv_weight_args), offsetof(b200rwkv_weight_args, n),\n'
                   '  offsetof(b200rwkv_weight_args, scale), offsetof(b200rwkv_weight_args, dst), offsetof(b200rwkv_weight_args, w),\n'
                   '  offsetof(b200rwkv_weight_args, out), offsetof(b200rwkv_weight_args, alpha), offsetof(b200rwkv_weight_args, rows),\n'
                   '  offsetof(b200rwkv_weight_args, blocks)); return 0; }\n')
    exe = tmp_path / "sz"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    O, G, W, L, K, WA = capi.Options, capi.GemmSeg, capi.WkvArgs, capi.LnArgs, capi.KeepArgs, capi.WeightArgs
    assert got == [C.sizeof(O), O.devices.offset, O.lora_st.offset, O.quant_layers.offset, C.sizeof(capi.Info),
                   C.sizeof(G), G.act.offset, G.lerp_xx.offset, G.out.offset,
                   C.sizeof(W), W.slot.offset, W.precision.offset, W.r.offset, W.nu.offset, W.layer0.offset, W.v_first.offset,
                   W.Dd.offset, W.out.offset,
                   W.nsnap.offset, W.snap_tok.offset, W.snap_rec.offset, W.snap_ld.offset, W.snap_off.offset,
                   C.sizeof(L), L.slot.offset, L.precision.offset, L.x_in.offset, L.parts.offset, L.n_mix.offset,
                   L.mix_out.offset, L.Dm.offset, L.V.offset, L.kernel_out.offset,
                   L.nsnap.offset, L.snap_tok.offset, L.snap_rec.offset, L.snap_ld.offset, L.snap_off.offset,
                   L.snap_head_out.offset,
                   C.sizeof(K), K.slot.offset, K.world.offset, K.shards.offset, K.keep.offset,
                   C.sizeof(WA), WA.n.offset, WA.scale.offset, WA.dst.offset, WA.w.offset, WA.out.offset, WA.alpha.offset,
                   WA.rows.offset, WA.blocks.offset]


def test_op_gemm_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_op_gemm checks every argument before its first CUDA call, so each refusal returns its status on a machine
    without a GPU: ERR_INVALID for malformed arguments, ERR_UNSUPPORTED for combinations the projection kernels do not run."""
    N, K, T = 64, 256, 4
    w = np.zeros((N, K), np.float16)
    x = np.zeros((1, T, K), np.float32)
    out = np.zeros((1, 16, N), np.float32)
    v = np.zeros((1, T, N), np.float32)

    def seg(**kw):
        s = capi.GemmSeg(N, K, capi.ptr(w), capi.ptr(x), None, capi.ACT_NONE, capi.OUT_F32, 0, None, None, None, N, capi.ptr(out))
        for k, val in kw.items():
            setattr(s, k, val)
        return s

    def call(segs=None, T=T, precision=0, quant=capi.QUANT_NONE, grid=0, launches=1, nseg=None):
        segs = [seg()] if segs is None else segs
        arr = (capi.GemmSeg * len(segs))(*segs)
        return capi.lib().b200rwkv_op_gemm(0, T, precision, quant, grid, launches, len(segs) if nseg is None else nseg, arr, None)

    INV, UNS = capi.ERR_INVALID, capi.ERR_UNSUPPORTED
    cases = {
        "null segment array": (capi.lib().b200rwkv_op_gemm(0, T, 0, 0, 0, 1, 1, None, None), INV),
        "no segment": (call(nseg=0), INV),
        "nine segments": (call([seg()] * 9), INV),
        "T = 0": (call(T=0), INV),
        "T = 129": (call(T=129), INV),
        "precision 2": (call(precision=2), INV),
        "negative grid": (call(grid=-1), INV),
        "no launch": (call(launches=0), INV),
        "quant_type 3": (call(quant=3), UNS),
        "precision 1 at T = 17": (call(T=17, precision=1), UNS),
        "precision 1 over Int8": (call(T=4, precision=1, quant=capi.QUANT_INT8), UNS),
        "null weight": (call([seg(w=None)]), INV),
        "null input": (call([seg(x=None)]), INV),
        "null output": (call([seg(out=None)]), INV),
        "N = 0": (call([seg(N=0)]), INV),
        "ldo < N": (call([seg(ldo=N - 1)]), INV),
        "unknown activation": (call([seg(act=7)]), INV),
        "unknown out_mode": (call([seg(out_mode=3)]), INV),
        "negative grp": (call([seg(out_mode=capi.OUT_A16, grp=-8)]), INV),
        "ddlerp without mu": (call([seg(out_mode=capi.OUT_LERP_A16, lerp_xx=capi.ptr(v), lerp_sx=capi.ptr(v))]), INV),
        "f16 output, N % 8": (call([seg(N=60, out_mode=capi.OUT_A16)]), UNS),
        "f16 output, grp % 8": (call([seg(out_mode=capi.OUT_A16, grp=12)]), UNS),
        "Int8, K % 128": (call([seg(K=200)], quant=capi.QUANT_INT8), UNS),
        "NF4, K % 128": (call([seg(), seg(K=96)], quant=capi.QUANT_NF4), UNS),
        "a bad second segment": (call([seg(), seg(ldo=0)]), INV),
    }
    for name, (got, want) in cases.items():
        assert got == want, name
    if not _has_gpu():                       # well-formed arguments reach the device, and there is none: no CPU fallback
        assert call() == capi.ERR_CUDA


def test_op_wkv_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_op_wkv checks every argument before its first CUDA call: ERR_INVALID for malformed arguments, ERR_STATE for a
    slot outside the pool, ERR_UNSUPPORTED for what the WKV kernels do not run."""
    H, S, T, Dd = 2, 4, 5, 64
    Cc = H * 64
    tok = np.zeros((T, Cc), np.float32)
    vec = np.zeros(Cc, np.float32)
    state = np.zeros((S, H, 64, 64), np.float32)
    out = np.zeros((16, Cc), np.uint16)
    d1 = np.zeros((T, Dd), np.float32)
    w2 = np.zeros((Cc, Dd), np.float16)
    P = capi.ptr

    def args(slots=(1, 3), counts=(2, 3), **kw):
        sl, cn = np.array(slots, np.int32), np.array(counts, np.int32)
        a = capi.WkvArgs(version=6, H=H, S=S, nslot=len(sl), slot=P(sl), count=P(cn), precision=0, r=P(tok), k=P(tok), v=P(tok),
                         g=P(tok), w=P(tok), u=P(vec), lnx_w=P(vec), lnx_b=P(vec), a=P(tok), k_k=P(vec), k_a=P(vec), r_k=P(vec),
                         nu=P(tok), layer0=1, v_first=P(tok), state=P(state), out=P(out))
        for k, val in kw.items():
            setattr(a, k, val)
        a._keep = (sl, cn)
        return a

    def call(a):
        return capi.lib().b200rwkv_op_wkv(0, C.byref(a))

    fold = dict(w=None, d1=P(d1), time_decay_w2=P(w2), decay_bias=P(vec), Dd=Dd)
    rec = np.zeros((3, 8 + H * 4096), np.float32)
    snap_toks = {n: np.array(t, np.int32) for n, t in (("ok", (0, 2, 4)), ("T", (0, 5, 1)), ("neg", (-1, 2, 4)), ("twice", (1, 3, 1)))}

    def snap(tok="ok", n=3, ld=8 + H * 4096, off=8, **kw):
        return {**dict(nsnap=n, snap_tok=P(snap_toks[tok]), snap_rec=P(rec), snap_ld=ld, snap_off=off), **kw}

    INV, UNS, STA = capi.ERR_INVALID, capi.ERR_UNSUPPORTED, capi.ERR_STATE
    cases = {
        "negative nsnap": (call(args(**snap(n=-1))), INV),
        "snapshots without tokens": (call(args(**snap(snap_tok=None))), INV),
        "snapshots without records": (call(args(**snap(snap_rec=None))), INV),
        "snapshot token T": (call(args(**snap("T"))), INV),
        "negative snapshot token": (call(args(**snap("neg"))), INV),
        "snapshot token twice": (call(args(**snap("twice"))), INV),
        "snap_ld < snap_off + H * 4096": (call(args(**snap(ld=4 + H * 4096))), INV),
        "negative snap_off": (call(args(**snap(off=-1))), INV),
        "snap_off past the int64 range": (call(args(**snap(off=2 ** 63 - 4))), INV),
        "snap_off % 4": (call(args(**snap(off=2))), INV),
        "snap_ld % 4": (call(args(**snap(ld=10 + H * 4096))), INV),
        "null arguments": (capi.lib().b200rwkv_op_wkv(0, None), INV),
        "version 4": (call(args(version=4)), UNS),
        "H = 0": (call(args(H=0)), INV),
        "H = 129": (call(args(H=129)), INV),
        "S = 0": (call(args(S=0)), INV),
        "no entry": (call(args(nslot=0)), INV),
        "more entries than slots": (call(args(slots=(0, 1, 2, 3, 4), counts=(1,) * 5)), INV),
        "null slot ids": (call(args(slot=None)), INV),
        "null counts": (call(args(count=None)), INV),
        "slot = S": (call(args(slots=(1, 4))), STA),
        "negative slot": (call(args(slots=(-1, 3))), STA),
        "duplicate slot": (call(args(slots=(3, 3))), INV),
        "count 0": (call(args(counts=(2, 0))), INV),
        "129 tokens": (call(args(counts=(64, 65))), INV),
        "precision 2": (call(args(precision=2)), INV),
        "precision 1 at T = 17": (call(args(counts=(8, 9), precision=1)), UNS),
        "null r": (call(args(r=None)), INV),
        "null g": (call(args(g=None)), INV),
        "null ln_x bias": (call(args(lnx_b=None)), INV),
        "null state": (call(args(state=None)), INV),
        "null out": (call(args(out=None)), INV),
        "v5 without u": (call(args(version=5, u=None)), INV),
        "v5 without w": (call(args(version=5, w=None)), INV),
        "v6 without w or fold": (call(args(w=None)), INV),
        "v6 without u": (call(args(u=None)), INV),
        "fold without decay_bias": (call(args(**dict(fold, decay_bias=None))), INV),
        "fold without d1": (call(args(**dict(fold, d1=None))), INV),
        "fold Dd = 0": (call(args(**dict(fold, Dd=0))), UNS),
        "fold Dd % 8": (call(args(**dict(fold, Dd=60))), UNS),
        "fold Dd = 136": (call(args(**dict(fold, Dd=136))), UNS),
        "v7 without a": (call(args(version=7, a=None)), INV),
        "v7 without w": (call(args(version=7, w=None)), INV),
        "v7 without r_k": (call(args(version=7, r_k=None)), INV),
        "v7 without v_first": (call(args(version=7, v_first=None)), INV),
        "v7 after layer 0 without nu": (call(args(version=7, layer0=0, nu=None)), INV),
    }
    for name, (got, want) in cases.items():
        assert got == want, name
    if not _has_gpu():                       # well-formed arguments reach the device, and there is none: no CPU fallback
        for ok in (args(), args(**fold), args(version=5), args(version=7, layer0=0), args(counts=(8, 8), precision=1),
                   args(**snap()), args(**snap(n=0, snap_tok=None, snap_rec=None))):
            assert call(ok) == capi.ERR_CUDA


def test_op_ln_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_op_ln checks every argument before its first CUDA call: ERR_INVALID for malformed arguments, ERR_STATE for a
    slot outside the pool, ERR_UNSUPPORTED for a front half or precision the kernels do not run."""
    Cc, S, T, Dm, V = 256, 4, 5, 32, 10
    tok = np.zeros((T, Cc), np.float32)
    vec = np.zeros(8 * Cc, np.float32)
    pool = np.zeros((S, Cc), np.float32)
    a16 = np.zeros((8, 32, Cc), np.uint16)
    ids = np.zeros(T, np.uint32)
    bad_ids = np.full(T, V, np.uint32)
    opt = np.zeros(2, np.int32)
    bad_opt = np.array([0, 3], np.int32)
    kern = np.zeros(3, np.int32)
    P = capi.ptr

    def args(slots=(1, 3), counts=(2, 3), **kw):
        sl, cn = np.array(slots, np.int32), np.array(counts, np.int32)
        a = capi.LnArgs(stage=capi.LN_MIX, C=Cc, S=S, nslot=len(sl), slot=P(sl), count=P(cn), option=P(opt), precision=0,
                        launches=1, x_in=P(tok), n_parts=1, n_gate=1, parts=P(tok), gates=P(tok), ln_w=P(vec), ln_b=P(vec),
                        shift_state=P(pool), n_mix=2, mu=P(vec), commit_src=P(tok), commit_dst=P(pool), hidden=P(tok),
                        x_out=P(tok), xx_out=P(tok), sx_out=P(tok), mix_out=P(a16), Dm=Dm, W1=P(a16), W2=P(a16), mu5=P(vec),
                        lora_out=P(a16), out5=P(a16), emb=P(a16), V=V, tokens=P(ids), head_out=P(a16), kernel_out=P(kern))
        for k, val in kw.items():
            setattr(a, k, val)
        a._keep = (sl, cn)
        return a

    def call(a):
        return capi.lib().b200rwkv_op_ln(0, C.byref(a))

    six = dict(stage=capi.LN_FRONT6, n_mix=1)
    rec = np.zeros((3, 8 + Cc), np.float32)
    snap_toks = {n: np.array(t, np.int32) for n, t in (("ok", (0, 2, 4)), ("T", (0, 5, 1)), ("neg", (-1, 2, 4)), ("twice", (1, 3, 1)))}

    def snap(tok="ok", n=3, ld=8 + Cc, off=8, **kw):
        return {**dict(nsnap=n, snap_tok=P(snap_toks[tok]), snap_rec=P(rec), snap_ld=ld, snap_off=off, snap_head_out=P(a16)), **kw}

    INV, UNS, STA = capi.ERR_INVALID, capi.ERR_UNSUPPORTED, capi.ERR_STATE
    cases = {
        "negative nsnap": (call(args(**snap(n=-1))), INV),
        "snapshots without tokens": (call(args(**snap(snap_tok=None))), INV),
        "snapshots without records": (call(args(**snap(snap_rec=None))), INV),
        "snapshot token T": (call(args(**snap("T"))), INV),
        "negative snapshot token": (call(args(**snap("neg"))), INV),
        "snapshot token twice": (call(args(**snap("twice"))), INV),
        "snap_ld < snap_off + C": (call(args(**snap(ld=4 + Cc))), INV),
        "negative snap_off": (call(args(**snap(off=-1))), INV),
        "snap_off past the int64 range": (call(args(**snap(off=2 ** 63 - 4))), INV),
        "snap_off % 4": (call(args(**snap(off=2))), INV),
        "snap_ld % 4": (call(args(**snap(ld=10 + Cc))), INV),
        "snapshots on the embed stage": (call(args(stage=capi.LN_EMBED, **snap())), INV),
        "snapshots over two launches": (call(args(launches=2, **snap())), INV),
        "ln_out snapshots without the commit": (call(args(stage=capi.LN_OUT, commit_src=None, commit_dst=None, **snap())), INV),
        "ln_out snapshots without snap_head_out": (call(args(stage=capi.LN_OUT, **snap(snap_head_out=None))), INV),
        "front half snapshots over two launches": (call(args(**six, launches=2, **snap())), INV),
        "null arguments": (capi.lib().b200rwkv_op_ln(0, None), INV),
        "stage 4": (call(args(stage=4)), INV),
        "C = 0": (call(args(C=0)), INV),
        "C % 64": (call(args(C=96)), INV),
        "C = 8256": (call(args(C=8256)), INV),
        "S = 0": (call(args(S=0)), INV),
        "S = 1025": (call(args(S=1025)), INV),
        "no entry": (call(args(nslot=0)), INV),
        "null slot ids": (call(args(slot=None)), INV),
        "null counts": (call(args(count=None)), INV),
        "slot = S": (call(args(slots=(1, 4))), STA),
        "negative slot": (call(args(slots=(-1, 3))), STA),
        "duplicate slot": (call(args(slots=(3, 3))), INV),
        "count 0": (call(args(counts=(2, 0))), INV),
        "129 tokens": (call(args(counts=(64, 65))), INV),
        "precision 2": (call(args(precision=2)), INV),
        "precision 1 at T = 17": (call(args(counts=(8, 9), precision=1)), UNS),
        "no launch": (call(args(launches=0)), INV),
        "17 launches": (call(args(launches=17)), INV),
        "null x_in": (call(args(x_in=None)), INV),
        "null ln_w": (call(args(ln_w=None)), INV),
        "nine parts": (call(args(n_parts=9)), INV),
        "negative n_gate": (call(args(n_gate=-1)), INV),
        "nine gates": (call(args(n_gate=9)), INV),
        "parts without buffer": (call(args(parts=None)), INV),
        "gates without buffer": (call(args(gates=None)), INV),
        "C / n_gate not whole": (call(args(n_gate=3)), INV),
        "commit_src alone": (call(args(commit_dst=None)), INV),
        "commit_dst alone": (call(args(commit_src=None)), INV),
        "n_mix 0": (call(args(n_mix=0)), INV),
        "n_mix 7": (call(args(n_mix=7)), INV),
        "null shift_state": (call(args(shift_state=None)), INV),
        "null mu": (call(args(mu=None)), INV),
        "null mix_out": (call(args(mix_out=None)), INV),
        "null xx_out": (call(args(xx_out=None)), INV),
        "in place with parts": (call(args(x_out=None)), INV),
        "front half, Dm 16": (call(args(**six, Dm=16)), UNS),
        "front half, C % 128": (call(args(**six, C=192, n_gate=0)), UNS),
        "front half, C = 4224": (call(args(**six, C=4224)), UNS),
        "front half, T = 17": (call(args(**six, counts=(8, 9))), UNS),
        "front half, two mixes": (call(args(**dict(six, n_mix=2))), INV),
        "front half without sx_out": (call(args(**six, sx_out=None)), INV),
        "front half without W1": (call(args(**six, W1=None)), INV),
        "front half without out5": (call(args(**six, out5=None)), INV),
        "ln_out without option": (call(args(stage=capi.LN_OUT, option=None)), INV),
        "ln_out without head": (call(args(stage=capi.LN_OUT, head_out=None)), INV),
        "ln_out, option 3": (call(args(stage=capi.LN_OUT, option=P(bad_opt))), INV),
        "embed without emb": (call(args(stage=capi.LN_EMBED, emb=None)), INV),
        "embed, V = 0": (call(args(stage=capi.LN_EMBED, V=0)), INV),
        "embed without tokens": (call(args(stage=capi.LN_EMBED, tokens=None)), INV),
        "embed, token V": (call(args(stage=capi.LN_EMBED, tokens=P(bad_ids))), INV),
        "embed without x_out": (call(args(stage=capi.LN_EMBED, x_out=None)), INV),
    }
    for name, (got, want) in cases.items():
        assert got == want, name
    if not _has_gpu():                       # well-formed arguments reach the device, and there is none: no CPU fallback
        for ok in (args(), args(x_out=None, n_parts=0), args(**six), args(**six, precision=1), args(stage=capi.LN_OUT),
                   args(stage=capi.LN_EMBED), args(counts=(60, 68), n_gate=8, n_parts=8), args(**snap()), args(**six, **snap()),
                   args(commit_src=None, commit_dst=None, **snap()), args(stage=capi.LN_OUT, **snap()),
                   args(stage=capi.LN_EMBED, **snap(n=0, snap_tok=None, snap_rec=None))):
            assert call(ok) == capi.ERR_CUDA


def test_op_keep_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_op_keep checks every argument before its first CUDA call: ERR_INVALID for malformed arguments, ERR_STATE for a
    slot outside the pool."""
    S, world, Vl = 4, 2, 5
    shards = np.zeros((world, 8, Vl), np.float32)
    keep = np.zeros((S, world * Vl), np.float32)
    P = capi.ptr

    def args(slots=(1, 3), counts=(2, 3), options=(capi.OPTION_FULL, capi.OPTION_LAST), **kw):
        sl, cn, op = np.array(slots, np.int32), np.array(counts, np.int32), np.array(options, np.int32)
        a = capi.KeepArgs(S=S, nslot=len(sl), slot=P(sl), count=P(cn), option=P(op), world=world, Vl=Vl, shards=P(shards),
                          keep=P(keep))
        for k, val in kw.items():
            setattr(a, k, val)
        a._keep = (sl, cn, op)
        return a

    def call(a):
        return capi.lib().b200rwkv_op_keep(0, C.byref(a))

    INV, STA = capi.ERR_INVALID, capi.ERR_STATE
    cases = {
        "null arguments": (capi.lib().b200rwkv_op_keep(0, None), INV),
        "world 0": (call(args(world=0)), INV),
        "world 9": (call(args(world=9)), INV),
        "Vl 0": (call(args(Vl=0)), INV),
        "world * Vl > 2^22": (call(args(world=8, Vl=(1 << 19) + 1)), INV),
        "S = 0": (call(args(S=0)), INV),
        "no entry": (call(args(nslot=0)), INV),
        "null slot ids": (call(args(slot=None)), INV),
        "null counts": (call(args(count=None)), INV),
        "slot = S": (call(args(slots=(1, 4))), STA),
        "negative slot": (call(args(slots=(-1, 3))), STA),
        "duplicate slot": (call(args(slots=(3, 3))), INV),
        "count 0": (call(args(counts=(2, 0))), INV),
        "129 tokens": (call(args(counts=(64, 65))), INV),
        "null options": (call(args(option=None)), INV),
        "option 3": (call(args(options=(capi.OPTION_LAST, capi.OPTION_SCORE))), INV),
        "null keep": (call(args(keep=None)), INV),
        "null shards with rows": (call(args(shards=None)), INV),
    }
    for name, (got, want) in cases.items():
        assert got == want, name
    if not _has_gpu():                       # well-formed arguments reach the device, and there is none: no CPU fallback
        none = (capi.OPTION_NONE, capi.OPTION_NONE)
        for ok in (args(), args(world=1), args(world=8, Vl=1 << 19), args(options=none, shards=None)):
            assert call(ok) == capi.ERR_CUDA


def test_op_weight_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_op_weight checks every argument of the chosen kind before its first CUDA call: ERR_INVALID for an unknown kind,
    a null buffer, an empty or oversized shape, or a sub-matrix outside its source."""
    w = np.zeros((8, 12), np.float16)
    lb, la = np.zeros((8, 3), np.float16), np.zeros((12, 3), np.float16)
    src = np.zeros((20, 30), np.float16)
    blocks = np.zeros(128 * 128, np.float16)
    dst = np.zeros(600, np.float32)
    P = capi.ptr
    L, F, D, R = capi.WEIGHT_LORA, capi.WEIGHT_F32, capi.WEIGHT_DECAY, capi.WEIGHT_REPACK

    def args(**kw):
        a = capi.WeightArgs(src=P(src), n=600, scale=1.0, bias=0.0, dst=P(dst), w=P(w), lora_b=P(lb), lora_a=P(la), out=8, in_=12,
                            r=3, alpha=0.5, rows=20, ld=30, n0=3, k0=5, N=17, K=25, blocks=P(blocks))
        for k, val in kw.items():
            setattr(a, k, val)
        return a

    def call(kind, a):
        return capi.lib().b200rwkv_op_weight(0, kind, C.byref(a))

    INV = capi.ERR_INVALID
    cases = {
        "null arguments": (capi.lib().b200rwkv_op_weight(0, L, None), INV),
        "kind -1": (call(-1, args()), INV),
        "kind 4": (call(4, args()), INV),
        "LoRA, null w": (call(L, args(w=None)), INV),
        "LoRA, null lora_b": (call(L, args(lora_b=None)), INV),
        "LoRA, null lora_a": (call(L, args(lora_a=None)), INV),
        "LoRA, out 0": (call(L, args(out=0)), INV),
        "LoRA, in 0": (call(L, args(in_=0)), INV),
        "LoRA, r 0": (call(L, args(r=0)), INV),
        "LoRA, r 4097": (call(L, args(r=4097)), INV),
        "LoRA, out * in > 2^31": (call(L, args(out=1 << 16, in_=(1 << 15) + 1)), INV),
        "f32, null src": (call(F, args(src=None)), INV),
        "f32, null dst": (call(F, args(dst=None)), INV),
        "f32, n 0": (call(F, args(n=0)), INV),
        "decay, n > 2^30": (call(D, args(n=(1 << 30) + 1)), INV),
        "decay, null dst": (call(D, args(dst=None)), INV),
        "repack, null src": (call(R, args(src=None)), INV),
        "repack, null blocks": (call(R, args(blocks=None)), INV),
        "repack, rows 0": (call(R, args(rows=0)), INV),
        "repack, ld 0": (call(R, args(ld=0)), INV),
        "repack, N 0": (call(R, args(N=0)), INV),
        "repack, K 0": (call(R, args(K=0)), INV),
        "repack, negative n0": (call(R, args(n0=-1)), INV),
        "repack, negative k0": (call(R, args(k0=-1)), INV),
        "repack, rows past the source": (call(R, args(N=18)), INV),
        "repack, columns past the source": (call(R, args(K=26)), INV),
    }
    for name, (got, want) in cases.items():
        assert got == want, name
    # a kind reads only its own members
    if not _has_gpu():                       # well-formed arguments reach the device, and there is none: no CPU fallback
        for kind, ok in ((L, args(src=None, dst=None, blocks=None)), (F, args(w=None, blocks=None)), (D, args(w=None, n=1)),
                         (R, args(w=None, dst=None, n0=0, k0=0, N=20, K=30))):
            assert call(kind, ok) == capi.ERR_CUDA


def test_c_host_program_links_and_calls_the_library(tmp_path):
    """A plain C host (no Python, no torch) includes include/b200rwkv.h, links libb200rwkv.so and calls the host-only entry
    points the Rust shim would call first (`Loader::info`, then `create`, which must fail loudly on a box without a GPU)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "ai00_server_b200")
    st = synth.make_st("tiny7", 0)
    stp = tmp_path / "m.st"
    stp.write_bytes(st.tobytes())
    src = tmp_path / "host.c"
    src.write_text(r'''
#include <stdio.h>
#include <stdlib.h>
#include "b200rwkv.h"
int main(int argc, char** argv) {
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
    uint8_t* buf = (uint8_t*)malloc((size_t)n);
    if (fread(buf, 1, (size_t)n, f) != (size_t)n) return 3;
    b200rwkv_info info;
    int32_t rc = b200rwkv_info_from_st(buf, (size_t)n, &info);
    printf("%d %d %d %d %d %d %d %d\n", rc, info.version, info.num_layer, info.num_emb, info.num_hidden, info.num_vocab, info.num_head, info.head_size);
    b200rwkv_engine* e = NULL;
    rc = b200rwkv_create(buf, (size_t)n, 0, 2, 32, 0, &e);
    printf("%d %s\n", rc, b200rwkv_last_error(NULL));
    if (e) b200rwkv_destroy(e);
    return 0;
}
''')
    exe = tmp_path / "host"
    subprocess.run([gcc, "-std=c99", "-Wall", "-I", os.path.join(root, "include"), str(src), "-o", str(exe), "-L", libdir, "-lb200rwkv",
                    "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe), str(stp)], check=True, capture_output=True, text=True).stdout.splitlines()
    s = synth.PRESETS["tiny7"]
    assert [int(x) for x in out[0].split()] == [0, 7, s.L, s.C, s.F, s.V, s.H, s.N]
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        rc, msg = out[1].split(" ", 1)
        assert int(rc) < 0 and "CUDA" in msg


def test_debug_fill_refuses_bad_arguments_without_a_gpu():
    """b200rwkv_debug_fills / debug_fill refuse a NULL engine, name or info with ERR_INVALID before any CUDA call, and write
    nothing (the engine-side refusals are in tests/test_gpu_resident_weights.py)."""
    lib = capi.lib()
    info = capi.FillInfo()
    info.kind = 77
    out = np.full(64, 0xAB, np.uint8)
    assert lib.b200rwkv_debug_fills(None, b"head.weight") == capi.ERR_INVALID
    assert lib.b200rwkv_debug_fills(None, None) == capi.ERR_INVALID
    for args in ((None, b"head.weight", 0, C.byref(info), capi.ptr(out), out.size), (None, None, 0, C.byref(info), None, 0),
                 (None, b"emb.weight", -1, None, capi.ptr(out), 0)):
        assert lib.b200rwkv_debug_fill(*args) == capi.ERR_INVALID
        assert "null argument" in lib.b200rwkv_last_error(None).decode()
    assert info.kind == 77 and np.all(out == 0xAB)


def test_fill_info_matches_the_header(tmp_path):
    """capi.FillInfo has the layout a C compiler gives b200rwkv_fill_info."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    fields = [n for n, _ in capi.FillInfo._fields_]
    src = tmp_path / "fi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200rwkv.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(b200rwkv_fill_info));\n' +
                   "".join(f'  printf("%zu\\n", offsetof(b200rwkv_fill_info, {n}));\n' for n in fields) + '  return 0; }\n')
    exe = tmp_path / "fi"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(capi.FillInfo)] + [getattr(capi.FillInfo, n).offset for n in fields]
    assert (capi.FILL_SEG, capi.FILL_VEC, capi.FILL_DECAY, capi.FILL_FOLD, capi.FILL_RAW, capi.FILL_INIT) == tuple(range(6))
    hdr = open(os.path.join(ROOT, "include", "b200rwkv.h")).read()
    for i, k in enumerate(("SEG", "VEC", "DECAY", "FOLD", "RAW", "INIT")):
        assert f"#define B200RWKV_FILL_{k} {i}\n" in hdr
    for i, k in enumerate(("BASE", "ADAPTER", "HEAD")):
        assert f"#define B200RWKV_PLAN_{k} {i}\n" in hdr
